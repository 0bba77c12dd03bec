// step_kernels.cuh -- the fiber half of System::step (system.cpp:482-492) on the device, one CTA per fiber:
//
//   FiberContainerFiniteDifference::step            (fcfd.cpp:292-302)  the fiber's [x(n); y(n); z(n); T(n)] block of the
//                                                                        solution -> AoS positions and the tension
//   FiberContainerFiniteDifference::repin_to_bodies (fcfd.cpp:308-316)  a bound fiber: delta = site - x_0 once, then
//                                                                        x_i + delta for every node
//   FiberContainerFiniteDifference::fiber_error_local (fcfd.cpp:79-89)  xs = (2 / length_) x D_1_0 on the repinned nodes,
//                                                                        max_i | ||xs_i|| - 1 | per fiber
//
// The fiber's nodes are staged in shared memory (3n doubles); D_1_0 is read from the class table through L1 / L2, only
// over the non-zero row range of each column (its finite-difference stencil), so no whole 128 KB matrix is staged.
// The per-fiber maximum is a fixed-shape tree of max operations: exact, so reproducible bit for bit.
//
// group_fiber_step_kernel is the same step of a rank-per-GPU member's own fibers, fused with the all-gather of its
// results: each new position and each per-fiber error is stored straight into the r_step piece of every member's group
// window (DESIGN.md §4), at its place among ALL fibers.  The values are those fiber_step_kernel writes, bit for bit:
// both kernels run one body (fiber_step) and differ only in where its outputs go.
#pragma once
#include "skb_internal.hpp" // StepItem

namespace skb {

constexpr int kStepThreads = 128;
constexpr int kStepMaxNodes = 128; // the device build's largest fiber (kBuildMaxNodes): 3n doubles of shared memory

// NaN wins: a fiber with a non-finite node reports a NaN error instead of hiding it
__device__ __forceinline__ double step_max(double a, double b) { return (a > b || a != a) ? a : b; }

// the outputs of fiber_step_kernel: its own buffers (r_out only FROM_SOLUTION)
struct StepOut {
    double *r_out, *err;
    __device__ __forceinline__ void pos(long long node, int k, double v) const { r_out[3 * node + k] = v; }
    __device__ __forceinline__ void error(double v) const { err[blockIdx.x] = v; }
};

// One fiber per CTA (blockIdx.x).  FROM_SOLUTION: in = the fibers' block of a solution vector (4 per node); the new AoS
// positions go to out.pos and the tensions to tension.  Otherwise in = AoS positions (3 per node), only the error is
// formed.  out.error: the fiber's max_i | ||xs_i|| - 1 |.  length: length_ per fiber of the launch.
template <bool FROM_SOLUTION, class Out>
__device__ __forceinline__ void fiber_step(const StepItem *__restrict__ items, const double *__restrict__ in,
                                           const double *__restrict__ class_mats,
                                           const int2 *__restrict__ class_ranges, const double *__restrict__ length,
                                           double *__restrict__ tension, const Out &out) {
    __shared__ double p[3 * kStepMaxNodes]; // x row | y row | z row
    __shared__ double wmax[kStepThreads / 32];
    const StepItem it = items[blockIdx.x];
    const int n = it.n;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        if (FROM_SOLUTION) {
            const double *xf = in + 4 * it.node;
            for (int k = 0; k < 3; ++k)
                p[k * n + i] = xf[k * n + i];
            tension[it.node + i] = xf[3 * n + i];
        } else {
            for (int k = 0; k < 3; ++k)
                p[k * n + i] = in[3 * (it.node + i) + k];
        }
    }
    __syncthreads();
    if (it.bound) {
        const double d0 = it.site[0] - p[0], d1 = it.site[1] - p[n], d2 = it.site[2] - p[2 * n];
        __syncthreads(); // every thread has read x_0 before node 0 moves
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            p[i] += d0;
            p[n + i] += d1;
            p[2 * n + i] += d2;
        }
        __syncthreads();
    }
    const double scale = 2.0 / length[blockIdx.x];
    const double *D = class_mats + it.d1;
    double e = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        if (FROM_SOLUTION)
            for (int k = 0; k < 3; ++k)
                out.pos(it.node + i, k, p[k * n + i]);
        const int2 r = class_ranges[it.rng + i];
        double s0 = 0.0, s1 = 0.0, s2 = 0.0;
        for (int j = r.x; j < r.y; ++j) {
            const double d = __ldg(D + (long long)i * n + j);
            s0 += p[j] * d;
            s1 += p[n + j] * d;
            s2 += p[2 * n + j] * d;
        }
        s0 *= scale, s1 *= scale, s2 *= scale;
        e = step_max(e, fabs(sqrt(s0 * s0 + s1 * s1 + s2 * s2) - 1.0));
    }
    for (int o = 16; o > 0; o >>= 1)
        e = step_max(e, __shfl_xor_sync(0xffffffffu, e, o));
    if ((threadIdx.x & 31) == 0)
        wmax[threadIdx.x >> 5] = e;
    __syncthreads();
    if (threadIdx.x == 0) {
        double m = wmax[0];
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
            m = step_max(m, wmax[w]);
        out.error(m);
    }
}

// r_out / tension receive the new AoS positions and the tensions (FROM_SOLUTION), err[blockIdx.x] the fiber's error
template <bool FROM_SOLUTION>
__global__ void __launch_bounds__(kStepThreads)
    fiber_step_kernel(const StepItem *__restrict__ items, const double *__restrict__ in,
                      const double *__restrict__ class_mats, const int2 *__restrict__ class_ranges,
                      const double *__restrict__ length, double *__restrict__ r_out, double *__restrict__ tension,
                      double *__restrict__ err) {
    fiber_step<FROM_SOLUTION>(items, in, class_mats, class_ranges, length, tension, StepOut{r_out, err});
}

constexpr int kStepMaxMembers = 16; // kMaxGroup (skb_internal.hpp), asserted where the group's window is laid out

// the outputs of group_fiber_step_kernel: r_step of every member's window, [3 per node of ALL fibers | 1 per fiber |
// 1 per fiber]: the new positions, the errors and (clamp not NULL) each fiber's minus_clamped flag, which a periphery
// shape's collision test needs of ALL fibers on every member
struct StepGather {
    double *r_step[kStepMaxMembers];
    int size;          // windows to store into
    long long n_fib;   // fiber nodes of ALL fibers: the errors start at r_step + 3 n_fib
    long long node0;   // the launch's first node among ALL fiber nodes
    int fiber0;        // the launch's first fiber among ALL fibers
    int n_fibers;      // ALL fibers: the flags start at r_step + 3 n_fib + n_fibers
    const int *clamp;  // per fiber among ALL fibers (NULL: no flags)
    __device__ __forceinline__ void pos(long long node, int k, double v) const {
        for (int m = 0; m < size; ++m)
            r_step[m][3 * (node0 + node) + k] = v;
    }
    __device__ __forceinline__ void error(double v) const {
        const int f = fiber0 + (int)blockIdx.x;
        for (int m = 0; m < size; ++m) {
            r_step[m][3 * n_fib + f] = v;
            if (clamp)
                r_step[m][3 * n_fib + n_fibers + f] = clamp[f] ? 1.0 : 0.0;
        }
    }
};

// a member's own fibers from its block of the solution (4 per own node): the tensions to `tension` (own nodes), the new
// positions and the errors into every window (defined in skb_step.cu, the one unit that launches it)
__global__ void __launch_bounds__(kStepThreads)
    group_fiber_step_kernel(const StepItem *__restrict__ items, const double *__restrict__ in,
                            const double *__restrict__ class_mats, const int2 *__restrict__ class_ranges,
                            const double *__restrict__ length, double *__restrict__ tension, const StepGather out);

} // namespace skb

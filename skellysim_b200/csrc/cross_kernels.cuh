// cross_kernels.cuh -- fiber <-> periphery in ONE geometry pass (sm_90a).
//
// System::apply_matvec visits every (fiber node i, periphery node j) pair twice per matvec: the fibers' Stokeslets act
// on the periphery nodes (fc.flow at r_all, src/core/system.cpp:299) and the periphery's stresslets act on the fiber
// nodes (shell.flow at r_fibbody, system.cpp:304,313-315).  Both kernels need d = x_i - x_j, r^2 and 1/r of the same
// pair (kernels.cu:29-40 and :62-72).  Evaluated separately that is 22 + 27 = 49 FP64 instructions per visited pair;
// sharing the geometry leaves 37:
//     forward  (stresslet of node j at fiber node i):    u_i += d (d.S_j.d) y^5          (kernels.cu:41-54)
//     reverse  (Stokeslet of fiber node i at node j):    u_j += y (h_i + d (h_i.d) y^2)   (kernels.cu:73-76; the
//                                                         displacement is -d, the two sign changes cancel)
// Work layout = pair_sym_kernel's (sym_kernels.cuh): the I side is a block of kSymThreads*T FIBER nodes held in registers
// (position, packed Stokeslet strength h, forward accumulators), the J side are groups of 32 PERIPHERY nodes staged by
// TMA (position + sym6 stresslet strength), walked as a ring inside each warp with the reverse accumulator travelling by
// shuffle; per-warp slabs, one barrier per stage, fixed-order sums -> bitwise reproducible.  Items are rectangles
// (fiber block I, periphery groups [g0, g1)); cross_reduce_kernel adds the forward partials of a block's items to the
// fiber rows and the reverse partials of all fiber blocks to the periphery rows.
#pragma once
#include "sym_kernels.cuh"

namespace skb {

constexpr int kCrossT = 4;    // fiber nodes per thread
constexpr int kCrossMinB = 3; // resident CTAs per SM
constexpr int kCrossBlock = kSymThreads * kCrossT;

struct CrossArgs {
    const double *r_fib;  // [n_fib_pad*3] fiber node positions (pads replicate the last node)
    const double *h;      // [n_fib_pad*3] packed (weighted) Stokeslet strengths, zero padded
    const double *r_sh;   // [n_sh_pad*3]  periphery node positions (pads replicate the last node)
    const double *s6;     // [n_sh_pad*6]  packed sym6 stresslet strengths, zero padded
    const SymItem *items; // (I = fiber block, periphery groups [g0, g1), slot, prow = I's row of P)
    double *P;            // [fiber blocks of this launch][n_sh_pad*3] reverse partials (Stokeslet sums at periphery nodes)
    double *F;            // [items][block*3] forward partials (stresslet sums at fiber nodes)
    long long n_sh_pad;
    long long node0;      // first fiber node of this launch (a group member evaluates its own fibers' rows)
    long long n_rows;     // fiber nodes of this launch; block I = nodes [node0 + I*block, ...), the tail beyond n_rows
                          // carries zero strength (other members' nodes / padding must not act on the periphery)
};

template <int T> struct CrossSmem {
    static constexpr int stage_bytes = kSymStageNodes * 72; // positions (24 B) + sym6 (48 B) per periphery node
    static constexpr int slab_doubles = kSymStageNodes * 3;
    static constexpr int slabs_bytes = 2 * (kSymThreads / 32) * slab_doubles * 8;
    static constexpr int bar_offset = kSymStages * stage_bytes + slabs_bytes;
    static constexpr int total_bytes = bar_offset + 2 * kSymStages * 8;
};

// T (fiber node, periphery record) pairs, both directions: 37 FP64 instructions per pair.
//   forward  uf_t += d co,          co = (d.S.d) y^5     (S = sxx, syy, szz, sxy+syx, sxz+szx, syz+szy of the record)
//   reverse  ur   += y (h_t + d (h_t.d) y^2)
template <int T>
__device__ __forceinline__ void cross_pairpairs(const double (&tx)[T], const double (&ty)[T], const double (&tz)[T],
                                                const double (&hx)[T], const double (&hy)[T], const double (&hz)[T],
                                                double rx, double ry, double rz, double sxx, double syy, double szz,
                                                double pxy, double pxz, double pyz, double (&ufx)[T], double (&ufy)[T],
                                                double (&ufz)[T], double &urx, double &ury, double &urz) {
    double dx[T], dy[T], dz[T], r2[T], y[T], q[T], co[T], v2[T], hr[T];
#pragma unroll
    for (int c = 0; c < T; ++c)
        dx[c] = tx[c] - rx;
#pragma unroll
    for (int c = 0; c < T; ++c)
        dy[c] = ty[c] - ry;
#pragma unroll
    for (int c = 0; c < T; ++c)
        dz[c] = tz[c] - rz;
#pragma unroll
    for (int c = 0; c < T; ++c)
        r2[c] = dx[c] * dx[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        r2[c] = fma(dy[c], dy[c], r2[c]);
#pragma unroll
    for (int c = 0; c < T; ++c)
        r2[c] = fma(dz[c], dz[c], r2[c]);
#pragma unroll
    for (int c = 0; c < T; ++c) {
        double y0;
        asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y0) : "d"(r2[c]));
        if (__double2hiint(r2[c]) < 0x00100000) // r == 0: the pair contributes exactly 0 in both directions
            y0 = 0.0;
        y[c] = y0;
    }
    // d.S.d, first half (shared operands: the record's components)
#pragma unroll
    for (int c = 0; c < T; ++c)
        co[c] = sxx * dx[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        co[c] = fma(pxy, dy[c], co[c]);
#pragma unroll
    for (int c = 0; c < T; ++c)
        co[c] = fma(pxz, dz[c], co[c]);
#pragma unroll
    for (int c = 0; c < T; ++c)
        v2[c] = syy * dy[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        v2[c] = fma(pyz, dz[c], v2[c]);
    // h.d
#pragma unroll
    for (int c = 0; c < T; ++c)
        hr[c] = hx[c] * dx[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        hr[c] = fma(hy[c], dy[c], hr[c]);
#pragma unroll
    for (int c = 0; c < T; ++c)
        hr[c] = fma(hz[c], dz[c], hr[c]);
    // 1/r: third-order Newton step on the seed (pair_kernels.cuh)
#pragma unroll
    for (int c = 0; c < T; ++c)
        r2[c] = r2[c] * y[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        r2[c] = fma(-r2[c], y[c], 1.0);
#pragma unroll
    for (int c = 0; c < T; ++c)
        q[c] = fma(0.375, r2[c], 0.5);
#pragma unroll
    for (int c = 0; c < T; ++c)
        q[c] = r2[c] * q[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        y[c] = fma(y[c], q[c], y[c]);
    // d.S.d, second half
#pragma unroll
    for (int c = 0; c < T; ++c)
        co[c] = co[c] * dx[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        q[c] = szz * dz[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        co[c] = fma(v2[c], dy[c], co[c]);
#pragma unroll
    for (int c = 0; c < T; ++c)
        co[c] = fma(q[c], dz[c], co[c]);
    // y^2 (both directions), y^5
#pragma unroll
    for (int c = 0; c < T; ++c)
        q[c] = y[c] * y[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        hr[c] = hr[c] * q[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        r2[c] = q[c] * q[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        r2[c] = r2[c] * y[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        co[c] = co[c] * r2[c];
#pragma unroll
    for (int c = 0; c < T; ++c) {
        ufx[c] = fma(dx[c], co[c], ufx[c]);
        ufy[c] = fma(dy[c], co[c], ufy[c]);
        ufz[c] = fma(dz[c], co[c], ufz[c]);
    }
#pragma unroll
    for (int c = 0; c < T; ++c) {
        urx = fma(y[c], fma(dx[c], hr[c], hx[c]), urx);
        ury = fma(y[c], fma(dy[c], hr[c], hy[c]), ury);
        urz = fma(y[c], fma(dz[c], hr[c], hz[c]), urz);
    }
}

template <int T, int MINB>
__global__ void __launch_bounds__(kSymThreads, MINB) pair_cross_kernel(const CrossArgs a) {
    using L = CrossSmem<T>;
    constexpr int kBlock = kSymThreads * T;
    constexpr int kWarps = kSymThreads / 32;
    extern __shared__ __align__(128) unsigned char smem[];
    double *slabs = reinterpret_cast<double *>(smem + kSymStages * L::stage_bytes);
    uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + L::bar_offset);
    uint64_t *empty_bar = full_bar + kSymStages;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const SymItem item = a.items[blockIdx.x];
    const int n_groups = item.g1 - item.g0;
    const int n_stages = (n_groups + kSymStageGroups - 1) / kSymStageGroups;

    auto issue_stage = [&](int k) {
        const int s = k % kSymStages;
        unsigned char *dst = smem + s * L::stage_bytes;
        const int g = item.g0 + k * kSymStageGroups;
        const int ng = (item.g1 - g) < kSymStageGroups ? (item.g1 - g) : kSymStageGroups;
        const uint32_t n_nodes = (uint32_t)ng * kSymGroup;
        mbar_arrive_expect_tx(&full_bar[s], n_nodes * 72);
        tma_bulk_g2s(dst, reinterpret_cast<const char *>(a.r_sh) + (size_t)g * kSymGroup * 24, n_nodes * 24, &full_bar[s]);
        tma_bulk_g2s(dst + kSymStageNodes * 24, reinterpret_cast<const char *>(a.s6) + (size_t)g * kSymGroup * 48,
                     n_nodes * 48, &full_bar[s]);
    };

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < kSymStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], kWarps);
        }
        mbar_fence_init();
        for (int k = 0; k < kSymPrefetch && k < n_stages; ++k)
            issue_stage(k);
    }
    double tx[T], ty[T], tz[T], hx[T], hy[T], hz[T], ufx[T], ufy[T], ufz[T];
#pragma unroll
    for (int t = 0; t < T; ++t) {
        const long long il = (long long)item.I * kBlock + t * kSymThreads + tid;
        const bool own = il < a.n_rows;
        const size_t i = (size_t)(a.node0 + (own ? il : a.n_rows - 1));
        tx[t] = __ldg(a.r_fib + 3 * i + 0), ty[t] = __ldg(a.r_fib + 3 * i + 1), tz[t] = __ldg(a.r_fib + 3 * i + 2);
        hx[t] = own ? __ldg(a.h + 3 * i + 0) : 0.0;
        hy[t] = own ? __ldg(a.h + 3 * i + 1) : 0.0;
        hz[t] = own ? __ldg(a.h + 3 * i + 2) : 0.0;
        ufx[t] = ufy[t] = ufz[t] = 0.0;
    }
    __syncthreads();

    for (int k = 0; k < n_stages; ++k) {
        const int s = k % kSymStages;
        if (tid == 0 && k + kSymPrefetch < n_stages) {
            const int kn = k + kSymPrefetch;
            if (kn >= kSymStages)
                mbar_wait(&empty_bar[kn % kSymStages], ((kn / kSymStages) - 1) & 1);
            issue_stage(kn);
        }
        const int g_first = item.g0 + k * kSymStageGroups;
        const int ng = (item.g1 - g_first) < kSymStageGroups ? (item.g1 - g_first) : kSymStageGroups;
        mbar_wait(&full_bar[s], (k / kSymStages) & 1);
        const double *ps = reinterpret_cast<const double *>(smem + s * L::stage_bytes);
        const double *ss = ps + kSymStageNodes * 3; // 6 doubles per node: 48 B stride, conflict-free for 64-bit loads
        double *slab_set = slabs + (k & 1) * kWarps * L::slab_doubles;
        double *my_slab = slab_set + warp * L::slab_doubles;
#pragma unroll 1
        for (int gi = 0; gi < ng; ++gi) {
            const int base = gi * kSymGroup;
            double urx = 0.0, ury = 0.0, urz = 0.0;
            double n_r[3], n_s[6];
            {
                const int idx = base + lane;
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    n_r[c] = ps[3 * idx + c];
#pragma unroll
                for (int c = 0; c < 6; ++c)
                    n_s[c] = ss[6 * idx + c];
            }
#pragma unroll 1
            for (int st = 0; st < 32; ++st) {
                const double rx = n_r[0], ry = n_r[1], rz = n_r[2];
                const double sxx = n_s[0], syy = n_s[1], szz = n_s[2], pxy = n_s[3], pxz = n_s[4], pyz = n_s[5];
                {
                    const int idx = base + ((lane + st + 1) & 31); // next step's record (the 33rd load is harmless)
#pragma unroll
                    for (int c = 0; c < 3; ++c)
                        n_r[c] = ps[3 * idx + c];
#pragma unroll
                    for (int c = 0; c < 6; ++c)
                        n_s[c] = ss[6 * idx + c];
                }
                cross_pairpairs<T>(tx, ty, tz, hx, hy, hz, rx, ry, rz, sxx, syy, szz, pxy, pxz, pyz, ufx, ufy, ufz, urx,
                                   ury, urz);
                const int from = (lane + 1) & 31;
                urx = __shfl_sync(0xffffffffu, urx, from);
                ury = __shfl_sync(0xffffffffu, ury, from);
                urz = __shfl_sync(0xffffffffu, urz, from);
            }
            my_slab[3 * (base + lane) + 0] = urx;
            my_slab[3 * (base + lane) + 1] = ury;
            my_slab[3 * (base + lane) + 2] = urz;
        }
        __syncwarp();
        if (lane == 0)
            mbar_arrive(&empty_bar[s]);
        __syncthreads();
        double *out = a.P + ((size_t)item.prow * a.n_sh_pad + (size_t)g_first * kSymGroup) * 3;
        for (int i = tid; i < ng * kSymGroup * 3; i += kSymThreads) {
            double v = slab_set[i];
#pragma unroll
            for (int w = 1; w < kWarps; ++w)
                v += slab_set[w * L::slab_doubles + i];
            out[i] = v;
        }
    }
    double *fo = a.F + (size_t)item.slot * kBlock * 3;
#pragma unroll
    for (int t = 0; t < T; ++t) {
        const int i = t * kSymThreads + tid;
        fo[3 * i + 0] = ufx[t];
        fo[3 * i + 1] = ufy[t];
        fo[3 * i + 2] = ufz[t];
    }
}

// u_fib[first_node + i] (+)= scale_dl * sum over the items of the node's block of F       (i < n_fib_rows)
__global__ void cross_reduce_fib_kernel(const double *__restrict__ F, const int *__restrict__ row_item_begin, int block,
                                        long long n_rows3, double scale_dl, int accumulate, double *__restrict__ u) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_rows3)
        return;
    const int b = (int)((i / 3) / block);
    const long long local = i - (long long)b * block * 3;
    double acc = 0.0;
    for (int it = row_item_begin[b]; it < row_item_begin[b + 1]; ++it)
        acc += F[(size_t)it * block * 3 + local];
    acc *= scale_dl;
    u[i] = accumulate ? u[i] + acc : acc;
}

// u_sh[j] (+)= scale_sl * sum over the fiber blocks of P[block][j]                         (j < n_sh)
__global__ void cross_reduce_shell_kernel(const double *__restrict__ P, int n_blocks, long long n_sh_pad, long long n_sh3,
                                          double scale_sl, int accumulate, double *__restrict__ u) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_sh3)
        return;
    double acc = 0.0;
    for (int b = 0; b < n_blocks; ++b)
        acc += P[(size_t)b * n_sh_pad * 3 + i];
    acc *= scale_sl;
    u[i] = accumulate ? u[i] + acc : acc;
}

} // namespace skb

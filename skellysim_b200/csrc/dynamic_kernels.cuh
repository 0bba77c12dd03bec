// dynamic_kernels.cuh -- the device half of System::dynamic_instability (dynamic_instability.cpp:25-194;
// skb_dynamic.cu, DESIGN.md §3.11): the per-fiber catastrophe and growth, the survivor scan, and the compaction of the
// fiber block with the nucleated fibers' straight lines appended.
#pragma once
#include "philox.cuh"

#include <cub/block/block_scan.cuh>
#include <cuda_runtime.h>

namespace skb {

constexpr int kDiThreads = 256;
constexpr int kDiScanThreads = 512; // (1024 caps the scan at 64 registers: it spills)
constexpr int kDiCompactThreads = 128;
// the scan carries (survivors, their nodes) in one 64-bit integer: survivors above bit 40, nodes below
constexpr int kDiCountShift = 40;
constexpr unsigned long long kDiNodeMask = (1ull << kDiCountShift) - 1;

// what the host decided once per call: the catastrophe thresholds exp(-dt f) and growth rates [not pinned, pinned]
struct DiRates {
    double thr[2], v[2], dt;
    unsigned long long seed, call;
};

// what the host reads back after the scan (one copy, with the keep and occupancy bytes behind it)
struct DiCounts {
    unsigned long long scan; // survivors << kDiCountShift | their nodes
    int n_bound;             // fibers bound before the catastrophe
    int pad;
};

// one thread per fiber f: the catastrophe draw (kept unless u > thr), the new length length + dt v (one rounded
// product and one rounded sum), the flat site of a bound survivor marked occupied, the bound fibers counted.
// fib[f] = (flat site or -1, plus_pinned)
__global__ void __launch_bounds__(kDiThreads)
    di_decide_kernel(int n, const int2 *__restrict__ fib, const double *__restrict__ length, DiRates r,
                     unsigned char *__restrict__ keep, double *__restrict__ len_new,
                     unsigned char *__restrict__ occupied, DiCounts *__restrict__ counts) {
    const int f = blockIdx.x * kDiThreads + threadIdx.x;
    int bound = 0;
    if (f < n) {
        const int2 a = fib[f];
        const double u = philox_uniform(r.seed, r.call, (uint32_t)f, kDiCatastrophe);
        const bool k = !(u > (a.y ? r.thr[1] : r.thr[0])); // (selects: an indexed parameter would go to local memory)
        keep[f] = k ? 1 : 0;
        len_new[f] = __dadd_rn(length[f], __dmul_rn(r.dt, a.y ? r.v[1] : r.v[0]));
        if (k && a.x >= 0)
            occupied[a.x] = 1;
        bound = a.x >= 0;
    }
    const int s = __syncthreads_count(bound);
    if (threadIdx.x == 0 && s)
        atomicAdd(&counts->n_bound, s); // an integer sum: the same whatever the order
}

// one block: the survivors in container order -- src[j] the input fiber of output fiber j, dst_off[j] its first node in
// the new block -- and counts->scan their total
__global__ void __launch_bounds__(kDiScanThreads)
    di_scan_kernel(int n, const unsigned char *__restrict__ keep, const long long *__restrict__ off,
                   int *__restrict__ src, long long *__restrict__ dst_off, DiCounts *__restrict__ counts) {
    using Scan = cub::BlockScan<unsigned long long, kDiScanThreads>;
    __shared__ typename Scan::TempStorage tmp;
    unsigned long long base = 0;
    for (int c0 = 0; c0 < n; c0 += kDiScanThreads) {
        const int f = c0 + threadIdx.x;
        const unsigned long long v =
            f < n && keep[f] ? (1ull << kDiCountShift) | (unsigned long long)(off[f + 1] - off[f]) : 0ull;
        unsigned long long ex, total;
        Scan(tmp).ExclusiveSum(v, ex, total);
        ex += base;
        if (v) {
            const long long j = (long long)(ex >> kDiCountShift);
            src[j] = f;
            dst_off[j] = (long long)(ex & kDiNodeMask);
        }
        base += total;
        __syncthreads(); // tmp is reused by the next chunk
    }
    if (threadIdx.x == 0)
        counts->scan = base;
}

// the nucleated fibers: n nodes of length L each; per body its rotation R (row-major) and centre c (12 doubles)
struct DiNew {
    int n;
    double L;
    long long node0; // first node of the first nucleated fiber (the survivors' nodes)
};

// one CTA per output fiber j: a survivor (j < n_surv) copies its nodes to their new offset and its new length; a
// nucleated fiber k = j - n_surv at pick (flat site, body) writes origin + u s_i, origin = c + R site_ref rounded as the
// step's nucleation sites are, u = (origin - c) / sqrt(|origin - c|^2), s_i = i (L / (n - 1)) and s_{n-1} = L
__global__ void __launch_bounds__(kDiCompactThreads)
    di_compact_kernel(int n_surv, const int *__restrict__ src, const long long *__restrict__ dst_off,
                      const long long *__restrict__ off, const double *__restrict__ r_old,
                      const double *__restrict__ len_new, const int2 *__restrict__ picks,
                      const double *__restrict__ site_ref, const double *__restrict__ frames, DiNew nw,
                      double *__restrict__ r_new, double *__restrict__ len_out) {
    const int j = blockIdx.x;
    if (j < n_surv) {
        const int f = src[j];
        const long long o = 3 * off[f], m = 3 * (off[f + 1] - off[f]), d = 3 * dst_off[j];
        for (long long i = threadIdx.x; i < m; i += kDiCompactThreads)
            r_new[d + i] = r_old[o + i];
        if (threadIdx.x == 0)
            len_out[j] = len_new[f];
        return;
    }
    const int k = j - n_surv;
    const int2 p = picks[k];
    const double *R = frames + 12 * (size_t)p.y, *c = R + 9, *s = site_ref + 3 * (size_t)p.x;
    double o[3], d[3];
    for (int a = 0; a < 3; ++a) {
        const double rs = __dadd_rn(__dadd_rn(__dmul_rn(R[3 * a], s[0]), __dmul_rn(R[3 * a + 1], s[1])),
                                    __dmul_rn(R[3 * a + 2], s[2]));
        o[a] = __dadd_rn(c[a], rs);
        d[a] = __dsub_rn(o[a], c[a]);
    }
    const double nrm =
        __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2])));
    const double u[3] = {__ddiv_rn(d[0], nrm), __ddiv_rn(d[1], nrm), __ddiv_rn(d[2], nrm)};
    const double step = __ddiv_rn(nw.L, (double)(nw.n - 1));
    double *x = r_new + 3 * (nw.node0 + (long long)k * nw.n);
    for (int i = threadIdx.x; i < nw.n; i += kDiCompactThreads) {
        const double si = i == nw.n - 1 ? nw.L : __dmul_rn((double)i, step);
        for (int a = 0; a < 3; ++a)
            x[3 * i + a] = __dadd_rn(o[a], __dmul_rn(u[a], si));
    }
    if (threadIdx.x == 0)
        len_out[j] = nw.L;
}

} // namespace skb

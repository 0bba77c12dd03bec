// sym_kernels.cuh -- Stokeslet self-interaction with Newton's third law (sm_90a).
//
// When the sources ARE the first n_src targets -- the fiber->fiber block that is ~90 % of the pairs of
// System::apply_matvec (r_all starts with the fiber nodes, src/core/system.cpp:284-299) -- the Oseen tensor is
// symmetric in the pair: G(x_i - x_j) = G(x_j - x_i).  d, r^2, 1/r and 1/r^2 (12 of the 22 FP64 instructions of a
// pair) can then serve both directions: 32 instructions per pair-of-pairs instead of 44.
//
// Layout of the work: nodes are cut into blocks of kSymThreads*T (the "I side": each thread keeps T nodes in registers:
// position, strength and the forward accumulators u_I += G f_J) and into GROUPS of 32 nodes (the "J side").  A work
// item is (block I, groups [g0, g1)) from block I's own first group onwards: the groups beyond block I are the strict
// upper triangle (both directions from one geometry pass); the groups of block I itself are the block diagonal, where
// the forward sums alone already cover every ordered pair (their reverse sums land in a part of P nobody reads).  The
// non-square remainder (targets beyond the sources) goes through pair_sum_kernel.  Items are as fine as one group (512*T/4 x 32 pairs), so the
// planner can hand out large items first and small ones last (cut_items, skb_sym.cu): the kernel's tail -- and the tail of
// every rank's share under multi-GPU sharding -- is a few stages, not one block pair.
// J groups are staged in shared memory by TMA, up to 4 groups per stage in a 4-stage ring; within a warp the 32 lanes
// walk a group as a ring: at step s lane l meets node (l + s) mod 32, and that node's reverse accumulator
// (u_J += G f_I) travels with it from lane to lane by one warp shuffle per step, so after 32 steps it is back home
// holding the sum over the warp's 32*T targets -- no cross-lane reduction tree.  Each warp parks its sums in its own
// shared-memory slab; once per stage the four slabs are added in a fixed order (bitwise reproducible) and written to
// the reverse partial P[row(I)][J nodes].  The final combination (sym_reduce_kernel) is a fixed-order sum.
#pragma once
#include <cstdint>
#include <type_traits>

#include "tma_ptx.cuh"

namespace skb {

constexpr int kSymThreads = 128;
constexpr int kSymT = 8;            // nodes of the I block per thread
constexpr int kSymMinB = 2;         // resident CTAs per SM
constexpr int kSymStages = 4;       // TMA ring depth (a stage is 6 KB)
constexpr int kSymPrefetch = kSymStages > 2 ? 2 : 1; // stages in flight ahead of the one being consumed
constexpr int kSymGroup = 32;       // nodes per J group (one ring)
constexpr int kSymStageGroups = 4;  // groups per stage
constexpr int kSymStageNodes = kSymGroup * kSymStageGroups;
constexpr int kSymGroupsPerBlock = kSymThreads * kSymT / kSymGroup;

struct SymItem {
    int I, g0, g1, slot; // I block, J groups [g0, g1) (from block I's own first group on), forward-partial slab index
    int prow, pad;       // row of P this item writes: index of I among the block rows owned by this part
};

struct SymArgs {
    const double *r;      // [n_pad*3] node positions, padded to a multiple of the block (pads replicate the last node)
    const double *f;      // [n_pad*3] packed Stokeslet strengths, zero padded
    const int *fid;       // [n_pad] fiber index of every node (EXCL kernels only)
    const SymItem *items; // [gridDim.x]
    double *P;            // [owned rows][n_pad*3]  reverse partials: P[prow(I)][node of J] = sum over targets in I
    double *F;            // [n_items][block*3] forward partials of each item
    long long n_pad;
    int nb;
};

template <int T> struct SymSmem {
    static constexpr int block = kSymThreads * T;
    static constexpr int stage_bytes = kSymStageNodes * 52; // positions + strengths (+ fiber ids) of one stage
    static constexpr int slab_doubles = kSymStageNodes * 3; // one warp's reverse sums of one stage
    static constexpr int slabs_bytes = 2 * (kSymThreads / 32) * slab_doubles * 8; // double-buffered
    static constexpr int bar_offset = kSymStages * stage_bytes + slabs_bytes;
    static constexpr int total_bytes = bar_offset + 2 * kSymStages * 8;
};

// T pair-of-pairs: targets (tx,ty,tz | strength hx,hy,hz) against ONE record (rx,ry,rz | strength gx,gy,gz).
// forward:  uf_t += y (g + d (g.d) y^2)      reverse:  ur += y (h_t + d (h_t.d) y^2)       d = x_t - x_rec
// (the reverse displacement is -d; the two sign changes cancel).  32 FP64 instructions per pair-of-pairs.
// EXCL (SURVEY.md 8f N3, opt-in): pairs whose two nodes belong to the same fiber contribute exactly 0 -- the fused form
// of FiberContainerFiniteDifference::flow's "all pairs, then subtract the fiber's own block"
// (fiber_container_finite_difference.cpp:203-210).  The fiber ids are compared in the integer pipe next to the r == 0
// rule and mask the same reciprocal-square-root seed: no FP64 instruction is added.
// REV = false: forward direction only (22 FP64 instructions per pair) -- the groups of block I itself, where the forward
// sums alone cover every ordered pair of the block diagonal.
template <int T, bool EXCL = false, bool REV = true>
__device__ __forceinline__ void stokeslet_pairpairs(const double (&tx)[T], const double (&ty)[T],
                                                    const double (&tz)[T], const double (&hx)[T],
                                                    const double (&hy)[T], const double (&hz)[T], double rx, double ry,
                                                    double rz, double gx, double gy, double gz, double (&ufx)[T],
                                                    double (&ufy)[T], double (&ufz)[T], double &urx, double &ury,
                                                    double &urz, const int (&tid)[T], int rid) {
    double dx[T], dy[T], dz[T], r2[T], y[T], q[T], fr[T], hr[T];
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
        if (__double2hiint(r2[c]) < 0x00100000 || (EXCL && tid[c] == rid))
            y0 = 0.0;
        y[c] = y0;
    }
#pragma unroll
    for (int c = 0; c < T; ++c)
        fr[c] = gx * dx[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        hr[c] = REV ? hx[c] * dx[c] : 0.0;
#pragma unroll
    for (int c = 0; c < T; ++c)
        fr[c] = fma(gy, dy[c], fr[c]);
#pragma unroll
    for (int c = 0; c < T; ++c)
        hr[c] = REV ? fma(hy[c], dy[c], hr[c]) : 0.0;
#pragma unroll
    for (int c = 0; c < T; ++c)
        fr[c] = fma(gz, dz[c], fr[c]);
#pragma unroll
    for (int c = 0; c < T; ++c)
        hr[c] = REV ? fma(hz[c], dz[c], hr[c]) : 0.0;
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
        y[c] = fma(y[c], q[c], y[c]); // 1/|d|
#pragma unroll
    for (int c = 0; c < T; ++c)
        q[c] = y[c] * y[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        fr[c] = fr[c] * q[c];
#pragma unroll
    for (int c = 0; c < T; ++c)
        hr[c] = REV ? hr[c] * q[c] : 0.0;
#pragma unroll
    for (int c = 0; c < T; ++c) {
        ufx[c] = fma(y[c], fma(dx[c], fr[c], gx), ufx[c]);
        ufy[c] = fma(y[c], fma(dy[c], fr[c], gy), ufy[c]);
        ufz[c] = fma(y[c], fma(dz[c], fr[c], gz), ufz[c]);
    }
    if constexpr (REV) {
#pragma unroll
        for (int c = 0; c < T; ++c) {
            urx = fma(y[c], fma(dx[c], hr[c], hx[c]), urx);
            ury = fma(y[c], fma(dy[c], hr[c], hy[c]), ury);
            urz = fma(y[c], fma(dz[c], hr[c], hz[c]), urz);
        }
    }
}

// The register cap is below the 256 that (kSymThreads, kSymMinB) allows: at 240 the two resident CTAs leave 1 024
// registers free in each of the SM's four sub-partitions -- room for the CTA of the background row streamer
// (stream_kernels.cuh), three warps of 32 registers.  (MINB, the residency the cap is chosen for, is not read here.)
constexpr int kSymMaxNReg = 240;
template <int T, int MINB, bool EXCL = false>
__global__ void __maxnreg__(kSymMaxNReg) pair_sym_kernel(const SymArgs a) {
    static_assert(T % 4 == 0, "the pair chains run in groups of 4");
    using L = SymSmem<T>;
    constexpr int kBlock = L::block;
    constexpr int kWarps = kSymThreads / 32;
    extern __shared__ __align__(128) unsigned char smem[];
    double *slabs = reinterpret_cast<double *>(smem + kSymStages * L::stage_bytes);
    uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + L::bar_offset);
    uint64_t *empty_bar = full_bar + kSymStages;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const SymItem item = a.items[blockIdx.x];
    const int n_groups = item.g1 - item.g0;
    const int n_stages = (n_groups + kSymStageGroups - 1) / kSymStageGroups;

    auto issue_stage = [&](int k) { // k-th stage of the item -> ring slot k % kSymStages
        const int s = k % kSymStages;
        unsigned char *dst = smem + s * L::stage_bytes;
        const int g = item.g0 + k * kSymStageGroups;
        const int ng = (item.g1 - g) < kSymStageGroups ? (item.g1 - g) : kSymStageGroups;
        const uint32_t bytes = (uint32_t)ng * kSymGroup * 24;
        const size_t off = (size_t)g * kSymGroup * 24;
        const uint32_t id_bytes = EXCL ? (uint32_t)ng * kSymGroup * 4 : 0u;
        mbar_arrive_expect_tx(&full_bar[s], 2 * bytes + id_bytes);
        tma_bulk_g2s(dst, reinterpret_cast<const char *>(a.r) + off, bytes, &full_bar[s]);
        tma_bulk_g2s(dst + kSymStageNodes * 24, reinterpret_cast<const char *>(a.f) + off, bytes, &full_bar[s]);
        if constexpr (EXCL)
            tma_bulk_g2s(dst + kSymStageNodes * 48, reinterpret_cast<const char *>(a.fid) + (size_t)g * kSymGroup * 4,
                         id_bytes, &full_bar[s]);
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
    // this thread's T nodes of block I: position, strength, forward accumulators
    double tx[T], ty[T], tz[T], hx[T], hy[T], hz[T], ufx[T], ufy[T], ufz[T];
    int tfid[T];
#pragma unroll
    for (int t = 0; t < T; ++t) {
        const size_t i = (size_t)item.I * kBlock + t * kSymThreads + tid;
        tfid[t] = EXCL ? __ldg(a.fid + i) : 0;
        tx[t] = __ldg(a.r + 3 * i + 0), ty[t] = __ldg(a.r + 3 * i + 1), tz[t] = __ldg(a.r + 3 * i + 2);
        hx[t] = __ldg(a.f + 3 * i + 0), hy[t] = __ldg(a.f + 3 * i + 1), hz[t] = __ldg(a.f + 3 * i + 2);
        ufx[t] = ufy[t] = ufz[t] = 0.0;
    }
    __syncthreads(); // barrier init visible

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
        const double *fs = ps + kSymStageNodes * 3;
        const int *ids = reinterpret_cast<const int *>(smem + s * L::stage_bytes + kSymStageNodes * 48);
        double *slab_set = slabs + (k & 1) * kWarps * L::slab_doubles; // double-buffered: one barrier per stage
        double *my_slab = slab_set + warp * L::slab_doubles;
        auto walk_group = [&](int gi, auto rev_tag) {
            constexpr bool REV = decltype(rev_tag)::value;
            const int base = gi * kSymGroup;
            double urx = 0.0, ury = 0.0, urz = 0.0;
            // the next step's record is loaded from shared memory before this step's chain (24 B stride: bank-conflict
            // free for 64-bit loads)
            double nrx, nry, nrz, ngx, ngy, ngz;
            int nid = 0;
            {
                const int idx = base + lane;
                nrx = ps[3 * idx + 0], nry = ps[3 * idx + 1], nrz = ps[3 * idx + 2];
                ngx = fs[3 * idx + 0], ngy = fs[3 * idx + 1], ngz = fs[3 * idx + 2];
                if constexpr (EXCL)
                    nid = ids[idx];
            }
#pragma unroll 1
            for (int st = 0; st < 32; ++st) {
                const double rx = nrx, ry = nry, rz = nrz, gx = ngx, gy = ngy, gz = ngz;
                const int rid = nid;
                {
                    const int idx = base + ((lane + st + 1) & 31); // (the 33rd load re-reads the first record: harmless)
                    nrx = ps[3 * idx + 0], nry = ps[3 * idx + 1], nrz = ps[3 * idx + 2];
                    ngx = fs[3 * idx + 0], ngy = fs[3 * idx + 1], ngz = fs[3 * idx + 2];
                    if constexpr (EXCL)
                        nid = ids[idx];
                }
                // chains in groups of 4: bounds the live temporaries
#pragma unroll
                for (int g0 = 0; g0 < T; g0 += 4) {
                    double ax[4], ay[4], az[4], bx[4], by[4], bz[4], cx[4], cy[4], cz[4];
                    int ti[4];
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        ti[c] = tfid[g0 + c];
                        ax[c] = tx[g0 + c], ay[c] = ty[g0 + c], az[c] = tz[g0 + c];
                        bx[c] = hx[g0 + c], by[c] = hy[g0 + c], bz[c] = hz[g0 + c];
                        cx[c] = ufx[g0 + c], cy[c] = ufy[g0 + c], cz[c] = ufz[g0 + c];
                    }
                    stokeslet_pairpairs<4, EXCL, REV>(ax, ay, az, bx, by, bz, rx, ry, rz, gx, gy, gz, cx, cy, cz, urx, ury,
                                                      urz, ti, rid);
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        ufx[g0 + c] = cx[c], ufy[g0 + c] = cy[c], ufz[g0 + c] = cz[c];
                }
                if constexpr (REV) {
                    // the record moves to lane - 1 for the next step; its accumulator goes with it
                    const int from = (lane + 1) & 31;
                    urx = __shfl_sync(0xffffffffu, urx, from);
                    ury = __shfl_sync(0xffffffffu, ury, from);
                    urz = __shfl_sync(0xffffffffu, urz, from);
                }
            }
            // after 32 steps lane l holds the finished sum of node base + l over this warp's 32*T targets
            // (forward-only groups park zeros: that part of P is never read)
            my_slab[3 * (base + lane) + 0] = urx;
            my_slab[3 * (base + lane) + 1] = ury;
            my_slab[3 * (base + lane) + 2] = urz;
        };
#pragma unroll 1
        for (int gi = 0; gi < ng; ++gi) {
            // groups of block I itself = the block diagonal: forward sums only (uniform over the CTA)
            if ((g_first + gi) / (kBlock / kSymGroup) == item.I)
                walk_group(gi, std::false_type());
            else
                walk_group(gi, std::true_type());
        }
        __syncwarp();
        if (lane == 0)
            mbar_arrive(&empty_bar[s]); // this warp is done reading the stage
        __syncthreads();                // all four slabs of this stage are complete
        // reverse partial of (I -> these groups): the four warps' sums in a fixed order, one coalesced write.
        // (the next stage's sums go to the other slab set; this set is rewritten only after the next barrier)
        double *out = a.P + ((size_t)item.prow * a.n_pad + (size_t)g_first * kSymGroup) * 3;
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

// Fixed-order combination for the symmetric path, one thread per velocity component of node `n` (block b):
//   u = (acc ? u : 0) + scale * ( sum_{owned I < b} P[prow(I)][n] + sum_{items of row b} F[item][n - b*block] )
// owned_rows[prow] = block row I of P's row prow (increasing); row b's own items cover the block diagonal as well
// (their groups start at block b itself), so nothing else is added.
__global__ void sym_reduce_kernel(const double *__restrict__ P, const double *__restrict__ F,
                                  const int *__restrict__ row_item_begin, const int *__restrict__ owned_rows,
                                  int n_owned, int block, long long n_pad, long long n_valid3, double scale,
                                  int accumulate, double *__restrict__ u) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; // component index 3*n + k
    if (i >= n_valid3)
        return;
    const long long node = i / 3;
    const int b = (int)(node / block);
    double acc = 0.0;
    for (int prow = 0; prow < n_owned && owned_rows[prow] < b; ++prow) // reverse partials of the rows above
        acc += P[((size_t)prow * n_pad) * 3 + i];
    const long long local = i - (long long)b * block * 3;
    for (int it = row_item_begin[b]; it < row_item_begin[b + 1]; ++it) // forward partials (empty for rows not owned)
        acc += F[(size_t)it * block * 3 + local];
    acc *= scale;
    u[i] = accumulate ? u[i] + acc : acc;
}

} // namespace skb

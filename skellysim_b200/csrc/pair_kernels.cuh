// pair_kernels.cuh -- sm_90a device code of the Stokeslet / stresslet all-pairs summation.
//
// What is computed (reference statements: SkellySim src/core/kernels.cu:57-77 Stokeslet, :24-55
// stresslet, driver :79-123; same math in src/core/kernels.cpp:11-40):
//   r = x_trg - x_src, rho = 1/|r| (0 when r == 0)
//   Stokeslet:  u += rho (f + r (f.r) rho^2)                       then u *= 1/(8 pi)
//   stresslet:  u += r (r.S.r) rho^5,  S = 3x3 from 9 doubles      then u *= -3/(8 pi)
//
// Design (written for the GPU, not a translation of the reference's 1-warp/1-target-per-thread kernel):
//   * FP64 vector pipe is the roofline (arithmetic intensity ~3e4 flop/B), so everything is shaped to
//     issue nothing but DFMA/DMUL/DADD on that pipe: 22 FP64 instr per Stokeslet pair, 27 per stresslet
//     pair.  The reciprocal square root is MUFU.RSQ64H (XU pipe, 2^-22 seed) + ONE third-order
//     Newton step (5 FP64 ops, rel. error ~1 ulp) instead of CUDA's ~12-instruction rsqrt().
//     The r == 0 rule is a predicated select on the seed (integer pipe), never a branch.
//   * register tiling: each consumer thread owns T targets (position + 3 accumulators in registers);
//     a source is broadcast from shared memory to the whole warp with 128-bit LDS, so shared-memory
//     traffic is 3 LDS.128 per source per warp against 22*T FP64 instructions.
//   * sources stream HBM/L2 -> shared memory with TMA bulk copies (cp.async.bulk, SASS UBLKCP) issued by
//     one elected lane two tiles ahead of use into a 4-stage ring guarded by full/empty mbarriers;
//     positions and strengths keep the caller's AoS layout, so a stage is two contiguous byte ranges and
//     no repacking pass is needed.
//   * the stresslet strength is pre-contracted once per matvec to its 6 symmetric combinations
//     (S only enters through r.S.r), cutting shared-memory bytes per source from 96 to 72.
//   * 2-D decomposition (target tile x source split) sized to the SM count; partial sums of the splits
//     are combined in a fixed order by a tiny second kernel -> bitwise run-to-run reproducible, no atomics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "tma_ptx.cuh"

namespace skb {

constexpr int kChainGroup = 4;      // independent pair chains evaluated stage-wise together when T >= 4
constexpr int kSrcTile = 128;       // sources per shared-memory stage
constexpr int kStages = 4;          // TMA ring depth
constexpr int kPrefetch = 2;        // tiles in flight ahead of the one being consumed (< kStages - 1)
constexpr int kCtaThreads = 128;    // 4 warps, one per SM sub-partition; every warp computes
constexpr int kMaxSplits = 256;

// the gradient kinds read the velocity kinds' packed strengths and write 10 outputs per target: d u_i / d x_j at
// 3 i + j, then the pressure (listener_gradient, skb_listener.cu)
enum Kind : int { kStokeslet = 0, kStresslet = 1, kStokesletGrad = 2, kStressletGrad = 3 };
template <int KIND> struct KindTraits;
// fdim: packed strengths per source; odim: outputs per target
template <> struct KindTraits<kStokeslet> { static constexpr int fdim = 3, odim = 3; };
template <> struct KindTraits<kStresslet> { static constexpr int fdim = 6, odim = 3; };  // sym6 combinations
template <> struct KindTraits<kStokesletGrad> { static constexpr int fdim = 3, odim = 10; };
template <> struct KindTraits<kStressletGrad> { static constexpr int fdim = 6, odim = 10; };

struct PairArgs {
    const double *r_src;   // [n_src_pad*3]   padded to a multiple of kSrcTile (pads replicate the last source)
    const double *f_src;   // [n_src_pad*fdim] padded with zeros
    const double *r_trg;   // [n_trg*3]
    double *partial;       // [n_splits][n_trg*3]
    long long n_trg;
    long long n_src;       // valid sources (the last tile is only walked up to here, rounded up to even)
    int n_src_tiles;       // ceil(n_src / kSrcTile)
    int tiles_per_split;   // source tiles handled by one blockIdx.y
    const int *src_fid;    // [n_src_pad] fiber id per source  (EXCL kernels only: same-fiber pairs contribute 0)
    const int *trg_fid;    // [n_trg]     fiber id per target
};

// ---------------------------------------------------------------------------------------------
// 1/sqrt(r2) in FP64 with the reference's r == 0 rule (inlined stage-wise in the *_chains routines below):
// MUFU.RSQ64H seed y0 (rel. err <= 2^-22.4), masked to 0 for r2 below the smallest normal (r2 == 0 and
// subnormal r2, which the seed instruction flushes), then y = y0 + y0 h, h = e (1/2 + 3/8 e), e = 1 - r2 y0^2:
// third-order, residual error ~(5/16) e^3 < 2^-64.  A zero seed stays exactly zero.
// ---------------------------------------------------------------------------------------------
// C independent (target, source) pair chains evaluated stage by stage, so a warp always has C FP64
// instructions in flight.  A single pair's chain is ~15 dependent FP64 instructions; issued back to back
// (what ptxas produces from a per-pair function under a tight register cap) it left the FP64 pipe idle
// for most of the DFMA latency.
// Stokeslet: 22 FP64 instructions per pair (kernels.cu:62-76);  outputs rinv y[c] and v = f + d (f.d) y^2.
// ---------------------------------------------------------------------------------------------
// EXCL: chains whose target and source carry the same fiber id (ti == si) contribute exactly 0 (sym_kernels.cuh).
template <int C, bool EXCL = false>
__device__ __forceinline__ void stokeslet_chains(const double (&tx)[C], const double (&ty)[C], const double (&tz)[C],
                                                 const double (&sx)[C], const double (&sy)[C], const double (&sz)[C],
                                                 const double (&fx)[C], const double (&fy)[C], const double (&fz)[C],
                                                 double (&y)[C], double (&vx)[C], double (&vy)[C], double (&vz)[C],
                                                 const int (&ti)[C], const int (&si)[C]) {
    // Instruction ORDER matters beyond dependencies: an FP64 instruction that reads 3 distinct 64-bit registers
    // occupies the pipe for 3 cycles instead of 2 (register-file read limit, scripts/ubench/fp64_ubench.cu) unless
    // one operand comes from the operand-reuse cache, i.e. the previous instruction read the same register in the
    // same operand slot.  Every 3-operand stage below therefore runs over the chains with one operand held fixed.
    double r2[C], fr[C], q[C];
#pragma unroll
    for (int c = 0; c < C; ++c)
        vx[c] = tx[c] - sx[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        vy[c] = ty[c] - sy[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        vz[c] = tz[c] - sz[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = vx[c] * vx[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = fma(vy[c], vy[c], r2[c]);
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = fma(vz[c], vz[c], r2[c]);
#pragma unroll
    for (int c = 0; c < C; ++c) {
        double y0;
        asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y0) : "d"(r2[c]));
        // r2 == 0 (or subnormal): the pair contributes exactly 0
        if (__double2hiint(r2[c]) < 0x00100000 || (EXCL && ti[c] == si[c]))
            y0 = 0.0;
        y[c] = y0;
    }
#pragma unroll
    for (int c = 0; c < C; ++c)
        fr[c] = fx[c] * vx[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        fr[c] = fma(fy[c], vy[c], fr[c]); // fy held fixed across the chains of one source
#pragma unroll
    for (int c = 0; c < C; ++c)
        fr[c] = fma(fz[c], vz[c], fr[c]);
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = r2[c] * y[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = fma(-r2[c], y[c], 1.0); // e = 1 - r2 y0^2
#pragma unroll
    for (int c = 0; c < C; ++c)
        q[c] = fma(0.375, r2[c], 0.5);
#pragma unroll
    for (int c = 0; c < C; ++c)
        q[c] = r2[c] * q[c]; // h = e (1/2 + 3/8 e)
#pragma unroll
    for (int c = 0; c < C; ++c)
        y[c] = fma(y[c], q[c], y[c]); // 1/|r| = y0 + y0 h   (2 distinct registers)
#pragma unroll
    for (int c = 0; c < C; ++c)
        q[c] = y[c] * y[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        q[c] = fr[c] * q[c]; // (f.d)/|r|^2
    // v_k = d_k q + f_k, walked so that consecutive instructions share f_k (within a row) or q (at the turns)
#pragma unroll
    for (int c = 0; c < C; ++c)
        vx[c] = fma(vx[c], q[c], fx[c]);
#pragma unroll
    for (int c = C - 1; c >= 0; --c)
        vy[c] = fma(vy[c], q[c], fy[c]);
#pragma unroll
    for (int c = 0; c < C; ++c)
        vz[c] = fma(vz[c], q[c], fz[c]);
}

// stresslet: 27 FP64 instructions per pair; s = (sxx, syy, szz, sxy+syx, sxz+szx, syz+szy), the -3 lives in the
// post-scale (kernels.cu:29-54).  Outputs d[c] and the scalar coefficient co[c] = (d.S.d)/|d|^5.
template <int C>
__device__ __forceinline__ void stresslet_chains(const double (&tx)[C], const double (&ty)[C], const double (&tz)[C],
                                                 const double (&sx)[C], const double (&sy)[C], const double (&sz)[C],
                                                 const double (&sxx)[C], const double (&syy)[C],
                                                 const double (&szz)[C], const double (&pxy)[C],
                                                 const double (&pxz)[C], const double (&pyz)[C], double (&dx)[C],
                                                 double (&dy)[C], double (&dz)[C], double (&co)[C]) {
    // same ordering rule as stokeslet_chains: 3-register stages keep one operand fixed across the chains
    double r2[C], y[C], v2[C], q[C];
#pragma unroll
    for (int c = 0; c < C; ++c)
        dx[c] = tx[c] - sx[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        dy[c] = ty[c] - sy[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        dz[c] = tz[c] - sz[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = dx[c] * dx[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = fma(dy[c], dy[c], r2[c]);
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = fma(dz[c], dz[c], r2[c]);
#pragma unroll
    for (int c = 0; c < C; ++c) {
        double y0;
        asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y0) : "d"(r2[c]));
        if (__double2hiint(r2[c]) < 0x00100000)
            y0 = 0.0;
        y[c] = y0;
    }
#pragma unroll
    for (int c = 0; c < C; ++c)
        co[c] = sxx[c] * dx[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        co[c] = fma(pxy[c], dy[c], co[c]);
#pragma unroll
    for (int c = 0; c < C; ++c)
        co[c] = fma(pxz[c], dz[c], co[c]);
#pragma unroll
    for (int c = 0; c < C; ++c)
        v2[c] = syy[c] * dy[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        v2[c] = fma(pyz[c], dz[c], v2[c]);
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = r2[c] * y[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = fma(-r2[c], y[c], 1.0);
#pragma unroll
    for (int c = 0; c < C; ++c)
        q[c] = fma(0.375, r2[c], 0.5);
#pragma unroll
    for (int c = 0; c < C; ++c)
        q[c] = r2[c] * q[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        y[c] = fma(y[c], q[c], y[c]); // 1/|r|
#pragma unroll
    for (int c = 0; c < C; ++c)
        co[c] = co[c] * dx[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        q[c] = szz[c] * dz[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        co[c] = fma(v2[c], dy[c], co[c]);
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = y[c] * y[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        co[c] = fma(q[c], dz[c], co[c]); // d.S.d
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = r2[c] * r2[c];
#pragma unroll
    for (int c = 0; c < C; ++c)
        r2[c] = r2[c] * y[c]; // 1/|r|^5
#pragma unroll
    for (int c = 0; c < C; ++c)
        co[c] = co[c] * r2[c];
}

// Two sources (a, b) against the thread's T targets, as groups of independent chains:
//   T == 1: one group of 2 chains (a, b);  T == 2: one group of 4 (2 targets x 2 sources);
//   T >= 4: per source, groups of 4 targets.
template <int T, bool EXCL = false>
__device__ __forceinline__ void stokeslet_two_sources(const double (&tx)[T], const double (&ty)[T],
                                                      const double (&tz)[T], const double (&sa)[3],
                                                      const double (&fa)[3], const double (&sb)[3],
                                                      const double (&fb)[3], double (&ux)[T], double (&uy)[T],
                                                      double (&uz)[T], const int (&tfid)[T], int ida, int idb) {
    if constexpr (T <= 2) {
        constexpr int C = 2 * T;
        double cx[C], cy[C], cz[C], sx[C], sy[C], sz[C], fx[C], fy[C], fz[C], y[C], vx[C], vy[C], vz[C];
        int ti[C], si[C];
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int t = c % T;
            const bool second = c >= T;
            ti[c] = tfid[t], si[c] = second ? idb : ida;
            cx[c] = tx[t], cy[c] = ty[t], cz[c] = tz[t];
            sx[c] = second ? sb[0] : sa[0], sy[c] = second ? sb[1] : sa[1], sz[c] = second ? sb[2] : sa[2];
            fx[c] = second ? fb[0] : fa[0], fy[c] = second ? fb[1] : fa[1], fz[c] = second ? fb[2] : fa[2];
        }
        stokeslet_chains<C, EXCL>(cx, cy, cz, sx, sy, sz, fx, fy, fz, y, vx, vy, vz, ti, si);
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int t = c % T;
            ux[t] = fma(y[c], vx[c], ux[t]);
            uy[t] = fma(y[c], vy[c], uy[t]);
            uz[t] = fma(y[c], vz[c], uz[t]);
        }
    } else {
        constexpr int G = kChainGroup;
#pragma unroll
        for (int src = 0; src < 2; ++src) {
#pragma unroll
            for (int g = 0; g < T / G; ++g) {
                double cx[G], cy[G], cz[G], sx[G], sy[G], sz[G], fx[G], fy[G], fz[G], y[G], vx[G], vy[G], vz[G];
                int ti[G], si[G];
#pragma unroll
                for (int c = 0; c < G; ++c) {
                    ti[c] = tfid[G * g + c], si[c] = src ? idb : ida;
                    cx[c] = tx[G * g + c], cy[c] = ty[G * g + c], cz[c] = tz[G * g + c];
                    sx[c] = src ? sb[0] : sa[0], sy[c] = src ? sb[1] : sa[1], sz[c] = src ? sb[2] : sa[2];
                    fx[c] = src ? fb[0] : fa[0], fy[c] = src ? fb[1] : fa[1], fz[c] = src ? fb[2] : fa[2];
                }
                stokeslet_chains<G, EXCL>(cx, cy, cz, sx, sy, sz, fx, fy, fz, y, vx, vy, vz, ti, si);
#pragma unroll
                for (int c = 0; c < G; ++c) {
                    ux[G * g + c] = fma(y[c], vx[c], ux[G * g + c]);
                    uy[G * g + c] = fma(y[c], vy[c], uy[G * g + c]);
                    uz[G * g + c] = fma(y[c], vz[c], uz[G * g + c]);
                }
            }
        }
    }
}

template <int T>
__device__ __forceinline__ void stresslet_two_sources(const double (&tx)[T], const double (&ty)[T],
                                                      const double (&tz)[T], const double (&sa)[3],
                                                      const double (&fa)[6], const double (&sb)[3],
                                                      const double (&fb)[6], double (&ux)[T], double (&uy)[T],
                                                      double (&uz)[T]) {
    if constexpr (T <= 2) {
        constexpr int C = 2 * T;
        double cx[C], cy[C], cz[C], sx[C], sy[C], sz[C], s0[C], s1[C], s2[C], s3[C], s4[C], s5[C];
        double dx[C], dy[C], dz[C], co[C];
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int t = c % T;
            const bool second = c >= T;
            cx[c] = tx[t], cy[c] = ty[t], cz[c] = tz[t];
            sx[c] = second ? sb[0] : sa[0], sy[c] = second ? sb[1] : sa[1], sz[c] = second ? sb[2] : sa[2];
            s0[c] = second ? fb[0] : fa[0], s1[c] = second ? fb[1] : fa[1], s2[c] = second ? fb[2] : fa[2];
            s3[c] = second ? fb[3] : fa[3], s4[c] = second ? fb[4] : fa[4], s5[c] = second ? fb[5] : fa[5];
        }
        stresslet_chains<C>(cx, cy, cz, sx, sy, sz, s0, s1, s2, s3, s4, s5, dx, dy, dz, co);
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int t = c % T;
            ux[t] = fma(dx[c], co[c], ux[t]);
            uy[t] = fma(dy[c], co[c], uy[t]);
            uz[t] = fma(dz[c], co[c], uz[t]);
        }
    } else {
        constexpr int G = kChainGroup;
#pragma unroll
        for (int src = 0; src < 2; ++src) {
#pragma unroll
            for (int g = 0; g < T / G; ++g) {
                double cx[G], cy[G], cz[G], sx[G], sy[G], sz[G], s0[G], s1[G], s2[G], s3[G], s4[G], s5[G];
                double dx[G], dy[G], dz[G], co[G];
#pragma unroll
                for (int c = 0; c < G; ++c) {
                    cx[c] = tx[G * g + c], cy[c] = ty[G * g + c], cz[c] = tz[G * g + c];
                    sx[c] = src ? sb[0] : sa[0], sy[c] = src ? sb[1] : sa[1], sz[c] = src ? sb[2] : sa[2];
                    s0[c] = src ? fb[0] : fa[0], s1[c] = src ? fb[1] : fa[1], s2[c] = src ? fb[2] : fa[2];
                    s3[c] = src ? fb[3] : fa[3], s4[c] = src ? fb[4] : fa[4], s5[c] = src ? fb[5] : fa[5];
                }
                stresslet_chains<G>(cx, cy, cz, sx, sy, sz, s0, s1, s2, s3, s4, s5, dx, dy, dz, co);
#pragma unroll
                for (int c = 0; c < G; ++c) {
                    ux[G * g + c] = fma(dx[c], co[c], ux[G * g + c]);
                    uy[G * g + c] = fma(dy[c], co[c], uy[G * g + c]);
                    uz[G * g + c] = fma(dz[c], co[c], uz[G * g + c]);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Velocity gradient and pressure of one source against the thread's T targets (the gradient kinds).  r = x_trg - x_src,
// y = 1/|r| with the velocity kernels' seed, Newton step and r == 0 rule (a coincident pair adds exactly 0 everywhere).
// The pressure output carries 2 (pressure numerator): with the velocity kind's post-scale s / eta it holds p / eta.
//   Stokeslet:  G_ij = d_i (f_j y^3 - 3 (f.r) y^5 r_j) - f_i r_j y^3 + delta_ij (f.r) y^3,  P = 2 (f.r) y^3
//   stresslet:  G_ij = d_i (h_j y^5 - 5 A y^7 r_j) + delta_ij A y^5,  h = grad_r A = 2 S_sym r,  A = r.S.r,
//               P = 2 A y^5 - (2/3) tr(S) y^3       (the -3 of the post-scale is kappa's)
// 10 accumulators per target; every output of a pair is an FMA chain into its accumulator.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double rsqrt_or_zero(double r2) {
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(r2));
    if (__double2hiint(r2) < 0x00100000)
        y = 0.0;
    const double e = fma(-r2 * y, y, 1.0);
    return fma(y, e * fma(0.375, e, 0.5), y);
}

template <int T>
__device__ __forceinline__ void stokeslet_grad_source(const double (&tx)[T], const double (&ty)[T],
                                                      const double (&tz)[T], const double (&s)[3],
                                                      const double (&f)[3], double (&g)[10][T]) {
#pragma unroll
    for (int t = 0; t < T; ++t) {
        const double d[3] = {tx[t] - s[0], ty[t] - s[1], tz[t] - s[2]};
        const double y = rsqrt_or_zero(fma(d[2], d[2], fma(d[1], d[1], d[0] * d[0])));
        const double y2 = y * y;
        const double y3 = y2 * y;
        const double a = fma(f[2], d[2], fma(f[1], d[1], f[0] * d[0])) * y3; // (f.r) / r^3
        const double b = 3.0 * a * y2;                                        // 3 (f.r) / r^5
        double p[3], q[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            q[j] = d[j] * y3;
            p[j] = fma(-d[j], b, f[j] * y3);
        }
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j)
                g[3 * i + j][t] = fma(-f[i], q[j], fma(d[i], p[j], g[3 * i + j][t]));
#pragma unroll
        for (int i = 0; i < 3; ++i)
            g[4 * i][t] += a;
        g[9][t] = fma(2.0, a, g[9][t]);
    }
}

template <int T>
__device__ __forceinline__ void stresslet_grad_source(const double (&tx)[T], const double (&ty)[T],
                                                      const double (&tz)[T], const double (&s)[3],
                                                      const double (&w)[6], double (&g)[10][T]) {
    // w = (sxx, syy, szz, sxy+syx, sxz+szx, syz+szy); tr(S) = w0 + w1 + w2
    const double tr23 = (2.0 / 3.0) * (w[0] + w[1] + w[2]);
#pragma unroll
    for (int t = 0; t < T; ++t) {
        const double d[3] = {tx[t] - s[0], ty[t] - s[1], tz[t] - s[2]};
        const double y = rsqrt_or_zero(fma(d[2], d[2], fma(d[1], d[1], d[0] * d[0])));
        const double y2 = y * y;
        const double y3 = y2 * y;
        const double y5 = y3 * y2;
        double h[3]; // grad_r (r.S.r)
        h[0] = fma(2.0 * w[0], d[0], fma(w[3], d[1], w[4] * d[2]));
        h[1] = fma(w[3], d[0], fma(2.0 * w[1], d[1], w[5] * d[2]));
        h[2] = fma(w[4], d[0], fma(w[5], d[1], 2.0 * w[2] * d[2]));
        const double A5 = 0.5 * fma(h[2], d[2], fma(h[1], d[1], h[0] * d[0])) * y5; // A / r^5
        const double c = 5.0 * A5 * y2;
        double v[3];
#pragma unroll
        for (int j = 0; j < 3; ++j)
            v[j] = fma(-c, d[j], h[j] * y5);
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j)
                g[3 * i + j][t] = fma(d[i], v[j], g[3 * i + j][t]);
#pragma unroll
        for (int i = 0; i < 3; ++i)
            g[4 * i][t] += A5;
        g[9][t] = fma(2.0, A5, fma(-tr23, y3, g[9][t]));
    }
}

// shared-memory footprint of the main kernel
template <int KIND, int T, bool EXCL = false> struct SmemLayout {
    static constexpr int fdim = KindTraits<KIND>::fdim;
    static constexpr int pos_stage_bytes = kSrcTile * 3 * 8;
    static constexpr int f_stage_bytes = kSrcTile * fdim * 8;
    static constexpr int id_stage_bytes = EXCL ? kSrcTile * 4 : 0;
    static constexpr int stage_bytes = pos_stage_bytes + f_stage_bytes + id_stage_bytes;
    static constexpr int trg_bytes = kCtaThreads * T * 3 * 8;
    static constexpr int bar_offset = kStages * stage_bytes + trg_bytes;
    static constexpr int total_bytes = bar_offset + 2 * kStages * 8;
};

// ---------------------------------------------------------------------------------------------
// Main kernel: grid = (target tiles, source splits), block = 4 warps, all of them compute.
// Lane 0 of warp 0 doubles as the TMA producer: before computing tile k it issues the bulk copies of tile
// k + kPrefetch into the ring slot that every warp released two tiles ago, so the wait on that slot's
// "empty" barrier never blocks in practice and no registers are spent on a dedicated producer warp.
// ---------------------------------------------------------------------------------------------
template <int KIND, int T, int MINB, bool EXCL = false>
__global__ void __launch_bounds__(kCtaThreads, MINB) pair_sum_kernel(const PairArgs a) {
    static_assert(!EXCL || KIND == kStokeslet, "fiber self-exclusion is a Stokeslet (fiber -> fiber) notion");
    using L = SmemLayout<KIND, T, EXCL>;
    constexpr int kTileT = kCtaThreads * T;
    extern __shared__ __align__(128) unsigned char smem[];
    double *trg_s = reinterpret_cast<double *>(smem + kStages * L::stage_bytes);
    uint64_t *full_bar = reinterpret_cast<uint64_t *>(smem + L::bar_offset);
    uint64_t *empty_bar = full_bar + kStages;

    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const long long t_base = (long long)blockIdx.x * kTileT;
    const int per_cta = a.tiles_per_split;
    const int first_tile = (int)blockIdx.y * a.tiles_per_split;
    int n_tiles = a.n_src_tiles - first_tile;
    n_tiles = n_tiles < per_cta ? n_tiles : per_cta;
    if (n_tiles < 0)
        n_tiles = 0;
    const char *gp = reinterpret_cast<const char *>(a.r_src) + (size_t)first_tile * L::pos_stage_bytes;
    const char *gf = reinterpret_cast<const char *>(a.f_src) + (size_t)first_tile * L::f_stage_bytes;

    auto issue_tile = [&](int k) {
        const int s = k % kStages;
        unsigned char *dst = smem + s * L::stage_bytes;
        mbar_arrive_expect_tx(&full_bar[s], L::stage_bytes);
        tma_bulk_g2s(dst, gp + (size_t)k * L::pos_stage_bytes, L::pos_stage_bytes, &full_bar[s]);
        tma_bulk_g2s(dst + L::pos_stage_bytes, gf + (size_t)k * L::f_stage_bytes, L::f_stage_bytes, &full_bar[s]);
        if constexpr (EXCL)
            tma_bulk_g2s(dst + L::pos_stage_bytes + L::f_stage_bytes,
                         reinterpret_cast<const char *>(a.src_fid) + (size_t)(first_tile + k) * L::id_stage_bytes,
                         L::id_stage_bytes, &full_bar[s]);
    };

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], kCtaThreads / 32);
        }
        mbar_fence_init();
        for (int k = 0; k < kPrefetch && k < n_tiles; ++k)
            issue_tile(k);
    }
    // coalesced load of this CTA's contiguous target block (AoS xyz) into shared memory: 128-bit loads when the
    // block starts 16-byte aligned (always, except for an odd-offset sub-range of a target list); the tail is
    // filled with the last valid target so no lane ever computes on garbage
    {
        long long n_valid = a.n_trg - t_base;
        n_valid = n_valid < kTileT ? n_valid : kTileT;
        const double *g = a.r_trg + 3 * t_base;
        const int n_dbl = (int)n_valid * 3;
        int done = 0;
        if ((reinterpret_cast<unsigned long long>(g) & 15ULL) == 0) {
            const int n_vec = n_dbl >> 1;
            const double2 *g2 = reinterpret_cast<const double2 *>(g);
            double2 *s2 = reinterpret_cast<double2 *>(trg_s);
            for (int i = tid; i < n_vec; i += kCtaThreads)
                s2[i] = __ldg(g2 + i);
            done = n_vec << 1;
        }
        for (int i = done + tid; i < kTileT * 3; i += kCtaThreads)
            trg_s[i] = (i < n_dbl) ? __ldg(g + i) : __ldg(g + (n_dbl - 3) + (i % 3));
    }
    __syncthreads(); // barrier init + target block visible to everyone

    constexpr int kOut = KindTraits<KIND>::odim;
    double tx[T], ty[T], tz[T], ux[T], uy[T], uz[T];
    double g[kOut][T]; // the gradient kinds' outputs (the velocity kinds use ux, uy, uz)
    int tfid[T];
#pragma unroll
    for (int t = 0; t < T; ++t) {
        const int i = t * kCtaThreads + tid;
        tfid[t] = (EXCL && t_base + i < a.n_trg) ? __ldg(a.trg_fid + t_base + i) : -1;
        tx[t] = trg_s[3 * i + 0];
        ty[t] = trg_s[3 * i + 1];
        tz[t] = trg_s[3 * i + 2];
        ux[t] = uy[t] = uz[t] = 0.0;
        if constexpr (kOut > 3)
#pragma unroll
            for (int o = 0; o < kOut; ++o)
                g[o][t] = 0.0;
    }

    for (int k = 0; k < n_tiles; ++k) {
        const int s = k % kStages;
        if (tid == 0 && k + kPrefetch < n_tiles) {
            const int kn = k + kPrefetch;
            if (kn >= kStages)
                mbar_wait(&empty_bar[kn % kStages], ((kn / kStages) - 1) & 1);
            issue_tile(kn);
        }
        mbar_wait(&full_bar[s], (k / kStages) & 1);
        const double2 *ps = reinterpret_cast<const double2 *>(smem + s * L::stage_bytes);
        const double2 *fs = reinterpret_cast<const double2 *>(smem + s * L::stage_bytes + L::pos_stage_bytes);
        // pairs of sources to walk in this tile (the padded tail of the last tile is skipped)
        long long left = a.n_src - (long long)(first_tile + k) * kSrcTile;
        const int jmax = left >= kSrcTile ? kSrcTile / 2 : (int)((left + 1) >> 1);
        // the stresslet's longer body gains from exposing the next sources' LDS early
        constexpr int kUnroll = (KIND == kStresslet && T <= 4) ? 2 : 1;
#pragma unroll kUnroll
        for (int j = 0; j < jmax; ++j) {
            // two sources per iteration: 48 B of positions = 3 x LDS.128 (warp-wide broadcast)
            const double2 p0 = ps[3 * j + 0], p1 = ps[3 * j + 1], p2 = ps[3 * j + 2];
            const double sa[3] = {p0.x, p0.y, p1.x}, sb[3] = {p1.y, p2.x, p2.y};
            if constexpr (KIND == kStokeslet) {
                const double2 f0 = fs[3 * j + 0], f1 = fs[3 * j + 1], f2 = fs[3 * j + 2];
                const double fa[3] = {f0.x, f0.y, f1.x}, fb[3] = {f1.y, f2.x, f2.y};
                int ida = 0, idb = 0;
                if constexpr (EXCL) {
                    const int2 id2 = reinterpret_cast<const int2 *>(smem + s * L::stage_bytes + L::pos_stage_bytes +
                                                                    L::f_stage_bytes)[j];
                    ida = id2.x, idb = id2.y;
                }
                stokeslet_two_sources<T, EXCL>(tx, ty, tz, sa, fa, sb, fb, ux, uy, uz, tfid, ida, idb);
            } else if constexpr (KIND == kStresslet) {
                const double2 f0 = fs[6 * j + 0], f1 = fs[6 * j + 1], f2 = fs[6 * j + 2];
                const double2 f3 = fs[6 * j + 3], f4 = fs[6 * j + 4], f5 = fs[6 * j + 5];
                const double fa[6] = {f0.x, f0.y, f1.x, f1.y, f2.x, f2.y};
                const double fb[6] = {f3.x, f3.y, f4.x, f4.y, f5.x, f5.y};
                stresslet_two_sources<T>(tx, ty, tz, sa, fa, sb, fb, ux, uy, uz);
            } else if constexpr (KIND == kStokesletGrad) {
                const double2 f0 = fs[3 * j + 0], f1 = fs[3 * j + 1], f2 = fs[3 * j + 2];
                const double fa[3] = {f0.x, f0.y, f1.x}, fb[3] = {f1.y, f2.x, f2.y};
                stokeslet_grad_source<T>(tx, ty, tz, sa, fa, g);
                stokeslet_grad_source<T>(tx, ty, tz, sb, fb, g);
            } else {
                const double2 f0 = fs[6 * j + 0], f1 = fs[6 * j + 1], f2 = fs[6 * j + 2];
                const double2 f3 = fs[6 * j + 3], f4 = fs[6 * j + 4], f5 = fs[6 * j + 5];
                const double fa[6] = {f0.x, f0.y, f1.x, f1.y, f2.x, f2.y};
                const double fb[6] = {f3.x, f3.y, f4.x, f4.y, f5.x, f5.y};
                stresslet_grad_source<T>(tx, ty, tz, sa, fa, g);
                stresslet_grad_source<T>(tx, ty, tz, sb, fb, g);
            }
        }
        __syncwarp();
        if (lane == 0)
            mbar_arrive(&empty_bar[s]);
    }

    double *out = a.partial + (size_t)blockIdx.y * (size_t)a.n_trg * kOut;
#pragma unroll
    for (int t = 0; t < T; ++t) {
        const long long i = t_base + t * kCtaThreads + tid;
        if (i < a.n_trg) {
            if constexpr (kOut == 3) {
                out[3 * i + 0] = ux[t];
                out[3 * i + 1] = uy[t];
                out[3 * i + 2] = uz[t];
            } else {
#pragma unroll
                for (int o = 0; o < kOut; ++o)
                    out[kOut * i + o] = g[o][t];
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Fixed-order combination of the source-split partials, post-scale, optional accumulate.
//   u[i] = (accumulate ? u[i] : 0) + scale * sum_s partial[s][i]
// ---------------------------------------------------------------------------------------------
__global__ void reduce_partials_kernel(const double *__restrict__ partial, double *__restrict__ u, long long n3,
                                       int n_splits, double scale, int accumulate) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n3)
        return;
    double acc = 0.0;
    for (int s = 0; s < n_splits; ++s)
        acc += partial[(size_t)s * n3 + i];
    acc *= scale;
    u[i] = accumulate ? u[i] + acc : acc;
}

// The same for FEW targets and MANY splits (the planner cuts 1e5 sources into ~1 000 splits when a call has a few
// hundred targets: the body rows of a rank): one thread per element then walks ~1 000 dependent loads (10 us).  Here a
// CTA owns 32 consecutive elements, its 16 warps take the splits round-robin (coalesced 256-byte loads, two independent
// running sums each), and the warps' sums are added in warp order: still a fixed order, bitwise reproducible.
constexpr int kReduceWideWarps = 16;
__global__ void __launch_bounds__(32 * kReduceWideWarps)
    reduce_partials_wide_kernel(const double *__restrict__ partial, double *__restrict__ u, long long n3, int n_splits,
                                double scale, int accumulate) {
    __shared__ double sh[kReduceWideWarps][33];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const long long i = (long long)blockIdx.x * 32 + lane;
    double a0 = 0.0, a1 = 0.0;
    if (i < n3) {
        int s = w;
        for (; s + kReduceWideWarps < n_splits; s += 2 * kReduceWideWarps) {
            a0 += partial[(size_t)s * n3 + i];
            a1 += partial[(size_t)(s + kReduceWideWarps) * n3 + i];
        }
        if (s < n_splits)
            a0 += partial[(size_t)s * n3 + i];
    }
    sh[w][lane] = a0 + a1;
    __syncthreads();
    if (w == 0 && i < n3) {
        double acc = 0.0;
#pragma unroll
        for (int k = 0; k < kReduceWideWarps; ++k)
            acc += sh[k][lane];
        acc *= scale;
        u[i] = accumulate ? u[i] + acc : acc;
    }
}

// ---------------------------------------------------------------------------------------------
// Strength packing (once per matvec, O(n_src)).
// ---------------------------------------------------------------------------------------------
// Stokeslet: copy + optional per-source weight (trapezoid quadrature weight of
// fiber_container_finite_difference.cpp:185-193) + zero pad.
__global__ void pack_sl_kernel(const double *__restrict__ f, const double *__restrict__ w, double *__restrict__ out,
                               long long n_src, long long n_pad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pad * 3)
        return;
    const long long s = i / 3;
    double v = 0.0;
    if (s < n_src) {
        v = f[i];
        if (w)
            v *= w[s];
    }
    out[i] = v;
}
// stresslet 9 -> sym6: (sxx, syy, szz, sxy+syx, sxz+szx, syz+szy)   (kernels.cu:41-49)
__global__ void pack_dl9_kernel(const double *__restrict__ f9, double *__restrict__ out, long long n_src,
                                long long n_pad) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_pad)
        return;
    double o[6] = {0, 0, 0, 0, 0, 0};
    if (s < n_src) {
        const double *f = f9 + 9 * s;
        o[0] = f[0];
        o[1] = f[4];
        o[2] = f[8];
        o[3] = f[1] + f[3];
        o[4] = f[2] + f[6];
        o[5] = f[5] + f[7];
    }
#pragma unroll
    for (int k = 0; k < 6; ++k)
        out[6 * s + k] = o[k];
}
// stresslet strength formed on the device: S = 2 eta n (x) rho  (periphery.cpp:68-71,
// body_container.cpp:296-302) contracted straight to sym6.  Products are formed exactly as the reference
// does (2*eta*n_a*rho_b, left to right) before the symmetric sums, so the result equals pack_dl9 of the
// host-formed f_dl bit for bit.
__global__ void pack_dl_normal_density_kernel(const double *__restrict__ nrm, const double *__restrict__ rho,
                                              double two_eta, double *__restrict__ out, long long n_src,
                                              long long n_pad) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_pad)
        return;
    double o[6] = {0, 0, 0, 0, 0, 0};
    if (s < n_src) {
        const double n0 = two_eta * nrm[3 * s + 0], n1 = two_eta * nrm[3 * s + 1], n2 = two_eta * nrm[3 * s + 2];
        const double r0 = rho[3 * s + 0], r1 = rho[3 * s + 1], r2 = rho[3 * s + 2];
        o[0] = n0 * r0;
        o[1] = n1 * r1;
        o[2] = n2 * r2;
        // no FMA contraction here: the host forms the 9 products separately, then kernels.cu:47-49 adds them
        o[3] = __dadd_rn(__dmul_rn(n0, r1), __dmul_rn(n1, r0));
        o[4] = __dadd_rn(__dmul_rn(n0, r2), __dmul_rn(n2, r0));
        o[5] = __dadd_rn(__dmul_rn(n1, r2), __dmul_rn(n2, r1));
    }
#pragma unroll
    for (int k = 0; k < 6; ++k)
        out[6 * s + k] = o[k];
}
// positions: copy + pad by replicating the last source (zero strength there => exact zero contribution)
__global__ void pad_positions_kernel(const double *__restrict__ r, double *__restrict__ out, long long n_src,
                                     long long n_pad) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pad * 3)
        return;
    const long long s = i / 3;
    out[i] = (s < n_src) ? r[i] : r[3 * (n_src - 1) + (i % 3)];
}

// ---------------------------------------------------------------------------------------------
// Pure DFMA throughput probe (roofline denominator measured on the box, SURVEY.md 8d).
// ---------------------------------------------------------------------------------------------
__global__ void dfma_probe_kernel(double *out, int iters, double a, double b) {
    double x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k)
        x[k] = threadIdx.x * 1e-9 + k;
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int k = 0; k < 8; ++k)
            x[k] = fma(x[k], a, b);
    }
    double s = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k)
        s += x[k];
    if (s == 12345.678)
        out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

} // namespace skb

// group_kernels.cuh -- the exchange steps of a multi-GPU matvec, written against PEER MEMORY (NVLink / NVSwitch
// loads and stores from inside kernels) instead of library collectives.
//
// A group is one skb_flow per GPU -- all in one process (skb_mflow: the shape the reference's "direct evaluators need
// a single rank" rule admits, src/core/system.cpp:618-623) or one per process (CUDA IPC, rank-per-GPU hosts).  Every
// member owns a WINDOW of device memory that all members can address; its layout is described at the declaration of
// skb::Group (skb_internal.hpp), whose steps (skb_group.cu, the only includer of this file) launch these kernels.
//
// One matvec = (1) PUSH: every member packs the strengths of ITS fibers / periphery rows once and stores them into
// all windows (the pack kernel and the all-gather are one kernel; 2.3 MB per member at 1e5 nodes); (2) flag barrier;
// (3) pair kernels on local memory only (TMA sources come from the member's own window); (4) flag barrier;
// (5) PULL: every member adds up the partial velocities of its own fiber rows (and, with the cross kernel, of its own
// periphery rows) from all windows (the reduce-scatter, fused with the accumulation into the velocity vector).
// The whole-vector operator adds one store of the member's partial link forces into every window before (2) and one
// rank-order sum of them after it.  A rank-per-GPU member's whole-vector calls (skb_flow_group_*) first store its own
// rows of the solution vector -- body rows, and for the preconditioner periphery rows -- into every window and meet at
// the rows phase, so that every member reads the complete x_bodies / x_shell from its own window.
#pragma once
#include <cuda_runtime.h>

#include "skb_internal.hpp" // kMaxGroup, kMaxRowPieces

namespace skb {

constexpr int kGroupPhases = 6;
constexpr int kRowsPhase = 4; // the exchange of a member's own solution rows (skb_flow_group_* whole-vector calls)
constexpr int kDotsPhase = 5; // the all-reduce of a solve's dot products (Group::reduce_dots)

struct GroupPushArgs {
    // own fibers: raw forces -> weighted, into rows [fa, fa + n_f) of every member's f_sl
    const double *fw;     // [n_f*3]
    const double *weight; // [n_fib] trapezoid weights of ALL fiber nodes (nullptr: 1)
    long long fa, n_f;
    // own periphery rows: density -> sym6 (2 eta n (x) rho) into rows [sa, sa + n_s) of f_shell, raw into x_shell
    const double *density; // [n_s*3]
    const double *normal;  // [n_shell*3] normals of ALL periphery nodes
    long long sa, n_s;
    double two_eta;
    int size;
    double *f_sl[kMaxGroup];
    double *f_shell[kMaxGroup];
    double *x_shell[kMaxGroup];
};

// pack + all-gather in one pass: every value is formed once and stored to `size` windows (coalesced per window)
__global__ void group_push_kernel(const GroupPushArgs a) {
    const long long nf3 = a.n_f * 3;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nf3 + a.n_s; i += stride) {
        if (i < nf3) {
            const long long node = a.fa + i / 3;
            double v = a.fw[i];
            if (a.weight)
                v *= a.weight[node];
            const long long o = 3 * a.fa + i;
            for (int m = 0; m < a.size; ++m)
                a.f_sl[m][o] = v;
        } else {
            const long long s = i - nf3, g = a.sa + s;
            // products formed exactly as the host does (2*eta*n_a*rho_b, then the symmetric sums): bit-identical to
            // pack_dl_normal_density_kernel / pack_dl9 of the host-formed f_dl (periphery.cpp:68-71)
            const double n0 = a.two_eta * a.normal[3 * g + 0], n1 = a.two_eta * a.normal[3 * g + 1],
                         n2 = a.two_eta * a.normal[3 * g + 2];
            const double r0 = a.density[3 * s + 0], r1 = a.density[3 * s + 1], r2 = a.density[3 * s + 2];
            double o6[6];
            o6[0] = n0 * r0;
            o6[1] = n1 * r1;
            o6[2] = n2 * r2;
            o6[3] = __dadd_rn(__dmul_rn(n0, r1), __dmul_rn(n1, r0));
            o6[4] = __dadd_rn(__dmul_rn(n0, r2), __dmul_rn(n2, r0));
            o6[5] = __dadd_rn(__dmul_rn(n1, r2), __dmul_rn(n2, r1));
            for (int m = 0; m < a.size; ++m) {
                double *d6 = a.f_shell[m] + 6 * g;
#pragma unroll
                for (int k = 0; k < 6; ++k)
                    d6[k] = o6[k];
                double *dx = a.x_shell[m] + 3 * g;
                dx[0] = r0, dx[1] = r1, dx[2] = r2;
            }
        }
    }
}

struct GroupFlagArgs {
    unsigned long long *flags[kMaxGroup]; // every member's flag array [kGroupPhases][kMaxGroup]
    int rank, size, phase;
    unsigned long long epoch;
    int do_signal, do_wait;
    unsigned long long timeout_cycles; // a peer that never arrives must not hang the GPU: give up and flag an error
};

// flags[kGroupPhases * kMaxGroup] of a window is the error word
__global__ void group_flag_kernel(const GroupFlagArgs a) {
    const int m = threadIdx.x;
    if (m >= a.size)
        return;
    if (a.do_signal) {
        __threadfence_system(); // everything this member stored before (earlier kernels of the stream included)
        volatile unsigned long long *p = a.flags[m] + a.phase * kMaxGroup + a.rank;
        *p = a.epoch;
    }
    if (a.do_wait) {
        volatile unsigned long long *q = a.flags[a.rank] + a.phase * kMaxGroup + m;
        const long long t0 = clock64();
        while (*q < a.epoch) {
            if ((unsigned long long)(clock64() - t0) > a.timeout_cycles) {
                a.flags[a.rank][kGroupPhases * kMaxGroup] = 1ULL + (unsigned long long)m; // who was missing
                break;
            }
            __nanosleep(200);
        }
        __threadfence_system();
    }
}

struct GroupPullArgs {
    const double *u_part[kMaxGroup]; // every member's partial velocities (u_part [n_fib*3] or u_part_shell [n_shell*3])
    int size;
    long long fa, n_f; // own fiber rows
    double *v;         // [n_f*3] (+)= sum over members, fixed order
    int accumulate;
};

// reduce-scatter fused with the accumulation: own rows only, members added in rank order (bitwise reproducible)
__global__ void group_pull_kernel(const GroupPullArgs a) {
    const long long n3 = a.n_f * 3;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n3)
        return;
    double acc = a.accumulate ? a.v[i] : 0.0;
    for (int m = 0; m < a.size; ++m)
        acc += __ldcv(a.u_part[m] + 3 * a.fa + i); // peer memory: never from a stale cache line
    a.v[i] = acc;
}

// ---- the bodies' link forces and torques of the whole-vector operator (BodyContainer, body_container.cpp:128-135) ----
// Every member sums the links of ITS bound fibers per body (body_sum_kernel); the partials [F (3 n_b) | L (3 n_b)] go
// into the member's slot of every window before flag barrier A, and after it every member adds up the slots of its own
// window in rank order -- the MPI_Allreduce of the reference, bitwise the same total on every member and run to run.
struct GroupFtStoreArgs {
    const double *f, *t; // [n_bodies*3] each: this member's partial forces / torques
    int n3;              // 3 n_bodies
    int size;
    double *slot[kMaxGroup]; // this member's slot [6 n_bodies] in every window
};

__global__ void group_ft_store_kernel(const GroupFtStoreArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2 * a.n3)
        return;
    const double v = i < a.n3 ? a.f[i] : a.t[i - a.n3];
    for (int m = 0; m < a.size; ++m)
        a.slot[m][i] = v;
}

struct GroupFtReduceArgs {
    const double *slots; // this member's window: slot m at slots + m * stride
    long long stride;    // 6 n_bodies
    int first, count;    // the slots to add, in this order
    int n3;
    double *f, *t; // [n_bodies*3] each: the totals
};

__global__ void group_ft_reduce_kernel(const GroupFtReduceArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 2 * a.n3)
        return;
    double acc = 0.0;
    for (int m = a.first; m < a.first + a.count; ++m)
        acc += __ldcv(a.slots + m * a.stride + i); // stored by peers: never from a stale cache line
    if (i < a.n3)
        a.f[i] = acc;
    else
        a.t[i - a.n3] = acc;
}

// ---- the all-reduce of a solve's dot products (skb_flow_group_solve_system_device) ----
// The ft_part pattern: every member stores its m partial dots into its slot of every window, meets its peers at the dots
// phase, and adds the slots of its own window in rank order, so every member holds bitwise the same sums.
struct GroupDotsStoreArgs {
    const double *v; // [m] this member's partials
    int m, size;
    double *slot[kMaxGroup]; // this member's slot in every window
};

__global__ void group_dots_store_kernel(const GroupDotsStoreArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.m)
        return;
    const double v = a.v[i];
    for (int k = 0; k < a.size; ++k)
        a.slot[k][i] = v;
}

__global__ void group_dots_reduce_kernel(const double *slots, long long stride, int first, int count, int m,
                                         double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m)
        return;
    double acc = 0.0;
    for (int k = first; k < first + count; ++k)
        acc += __ldcv(slots + k * stride + i); // stored by peers: never from a stale cache line
    out[i] = acc;
}

// ---- a member's own rows of the solution vector (skb_flow_group_* whole-vector calls) ----
// The member's body rows are its local vector's body part, compacted in ascending global order; the piece table maps
// them onto the body part of the whole vector: piece p covers local entries [local, local + len) and body-part entries
// [body, body + len) (RowPieces, skb_internal.hpp: at most kMaxRowPieces, built when the body operators are set).
struct RowPiecesDev {
    long long local[kMaxRowPieces], body[kMaxRowPieces], len[kMaxRowPieces];
    int n;
    long long total; // sum of len
};

// the body-part offset of local entry i (the pieces ascend; unrolled over the table, so it stays in registers)
__device__ __forceinline__ long long row_piece_offset(const RowPiecesDev &p, long long i) {
    long long lo = p.local[0], bo = p.body[0];
#pragma unroll
    for (int k = 1; k < kMaxRowPieces; ++k)
        if (k < p.n && p.local[k] <= i)
            lo = p.local[k], bo = p.body[k];
    return bo + (i - lo);
}

struct GroupRowsStoreArgs {
    RowPiecesDev pieces;
    const double *body;  // [pieces.total] the own body rows of the local vector
    const double *shell; // [n_shell3] the own periphery rows (3 per row), NULL: none stored
    long long shell_off, n_shell3; // -> x_shell entries [shell_off, shell_off + n_shell3)
    int size;
    double *x_body[kMaxGroup];
    double *x_shell[kMaxGroup];
};

// the own rows into every window: body rows scattered to their place in x_body, periphery rows into x_shell
__global__ void group_rows_store_kernel(const GroupRowsStoreArgs a) {
    const long long nb = a.pieces.total, n = nb + a.n_shell3;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        if (i < nb) {
            const double v = a.body[i];
            const long long o = row_piece_offset(a.pieces, i);
            for (int m = 0; m < a.size; ++m)
                a.x_body[m][o] = v;
        } else {
            const long long s = i - nb;
            const double v = a.shell[s];
            for (int m = 0; m < a.size; ++m)
                a.x_shell[m][a.shell_off + s] = v;
        }
    }
}

struct GroupRowsCompactArgs {
    RowPiecesDev pieces;
    const double *full; // a body output in the whole body layout
    double *local;      // [pieces.total] the member's own rows of it
};

__global__ void group_rows_compact_kernel(const GroupRowsCompactArgs a) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.pieces.total)
        a.local[i] = a.full[row_piece_offset(a.pieces, i)];
}

} // namespace skb

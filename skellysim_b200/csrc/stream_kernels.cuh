// stream_kernels.cuh -- the BACKGROUND row streamer: y = A x for a row-major FP64 matrix, built to run BESIDE the
// FP64-bound pair kernels instead of after them.
//
// Why: the periphery's dense operator (Periphery::matvec, SkellySim src/core/periphery.cpp:38-47) reads 8 B per FMA -- it
// is bound by HBM and leaves the FP64 pipe idle; pair_sym_kernel is bound by the FP64 pipe and leaves HBM idle.  Run one
// after the other, the dense operator's time adds to the matvec's.  The classic GEMV (dense_gemv_kernel: 256 threads, all
// warps resident) cannot share an SM with the symmetric kernel, whose two CTAs held the whole register file.  This
// kernel can: ONE CTA of three warps x 32 registers per SM (a producer warp and two consumer warps).  The register file
// is split over the SM's four sub-partitions (16 384 registers each); pair_sym_kernel is capped at 240 registers, so its
// two CTAs (one warp per sub-partition each) leave 1 024 registers per sub-partition free -- exactly one 32-register
// warp each.  The matrix is moved by the TMA engine, not by threads --
//   * five lanes of the producer warp post 1-D bulk copies (cp.async.bulk, SASS UBLKCP): 4 rows x 512 columns of A plus
//     the 512 matching entries of x (L2 resident) = 20 KB per stage into a 5-stage ring, 4 stages (64 KB of A) ahead of
//     use: more than HBM latency x bandwidth per SM, so the ring keeps the SM's share of the bandwidth in flight with
//     no warp waiting on a load instruction (a first version read x with LDG: every stage then waited one L2 latency);
//   * the 64 consumer threads consume a stage with 20 LDS.128 + 32 DFMA each -- 4 % of the SM's FP64 issue slots while
//     it runs, 0.3 % of the symmetric kernel's total;
//   * the bulk copies carry an L2 evict-first policy: 2.6 GB of read-once matrix must not evict the 4.6 MB of node
//     records the pair kernels stream from L2.
// bench.py's `overlap` leg times the matvec with this kernel beside the pair kernels against the GEMV after them.
// Rows are handed out in groups of 4 by a ticket counter (first group static); a row's sum is accumulated in a fixed
// thread -> column mapping and a fixed reduction tree, so results are bitwise reproducible whatever the ticket order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "tma_ptx.cuh"

namespace skb {

constexpr int kStreamConsumers = 64;                 // two consumer warps
constexpr int kStreamThreads = kStreamConsumers + 32; // + the producer warp (five lanes active)
constexpr int kStreamRows = 4;     // rows per group (x is re-used 4 times per load)
constexpr int kStreamCols = 512;   // columns per stage (a multiple of 128)
constexpr int kStreamStages = 5;
constexpr int kStreamMaxNReg = 32; // registers per thread: fits beside pair_sym_kernel (see above)
constexpr int kStreamRowBytes = kStreamCols * 8;
constexpr int kStreamStageBytes = (kStreamRows + 1) * kStreamRowBytes; // rows of A, then the segment of x
// ring | full + empty barriers | (group, chunk) of every stage | cross-warp sums
constexpr int kStreamBarOffset = kStreamStages * kStreamStageBytes;
constexpr int kStreamMetaOffset = kStreamBarOffset + 2 * kStreamStages * 8;
constexpr int kStreamRedOffset = kStreamMetaOffset + kStreamStages * 8;
constexpr int kStreamSmemBytes = kStreamRedOffset + 2 * kStreamRows * 8;

struct StreamArgs {
    const double *A; // [n_rows][n_cols] row-major, n_cols even (every row 16-byte aligned)
    const double *x; // [n_cols], 16-byte aligned
    double *y;       // [n_rows]
    long long n_rows, n_cols;
    unsigned long long *next_group; // ticket counter, zero at launch
};

// defined in skb_dense.cu, the one translation unit that launches it (prepare_device in skb_runtime.cu sets its
// attributes)
__global__ void __maxnreg__(kStreamMaxNReg) dense_stream_kernel(const StreamArgs a);

} // namespace skb

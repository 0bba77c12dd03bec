// skb_dense.cu -- the periphery's dense operators (Periphery::matvec / apply_preconditioner,
// SkellySim src/core/periphery.cpp:21-47) as an HBM-bound row-major GEMV on H100.  include/skelly_b200_dense.h.
#include "skb_internal.hpp"
#include "stream_kernels.cuh"
#include "../../include/skelly_b200_dense.h"

#include <algorithm>
#include <cstdint>
#include <memory>
#include <vector>

using namespace skb;

namespace {

// 128-bit streaming load of the matrix (read once, keep it out of L1)
__device__ __forceinline__ double2 ldg_stream(const double2 *p) {
    double2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
    return v;
}

// y[r] = sum_c A[r][c] x[c] (+ v[r]).  One warp per row, rows strided over the grid; each lane walks the row in
// 16-byte pieces (512 B per warp-load, fully coalesced) with kUnroll independent loads in flight; x (<= 240 KB)
// lives in L1/L2.  Per-lane partial sums are combined by a fixed shuffle tree: bitwise reproducible.
constexpr int kGemvUnroll = 8;
__global__ void __launch_bounds__(256) dense_gemv_kernel(const double *__restrict__ A, const double *__restrict__ x,
                                                         const double *__restrict__ v, double *__restrict__ y,
                                                         long long n_rows, long long n_cols, int vec_ok,
                                                         unsigned long long *__restrict__ next_row) {
    const int lane = threadIdx.x & 31;
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
    // rows are handed out dynamically (18 000 rows over ~9 500 warps would otherwise leave a 2-vs-1 tail); the row a
    // warp gets does not change how that row is summed, so results stay bitwise reproducible.  The first row is
    // static, the ticket for the following one is drawn before the current row is streamed.
    long long r = warp;
    while (r < n_rows) {
        unsigned long long ticket = 0;
        if (lane == 0)
            ticket = atomicAdd(next_row, 1ULL);
        const long long r_next = n_warps + (long long)__shfl_sync(0xffffffffu, ticket, 0);
        const double *row = A + r * n_cols;
        double acc[kGemvUnroll];
#pragma unroll
        for (int u = 0; u < kGemvUnroll; ++u)
            acc[u] = 0.0;
        long long c = 0;
        if (vec_ok) {
            const double2 *row2 = reinterpret_cast<const double2 *>(row);
            const double2 *x2 = reinterpret_cast<const double2 *>(x);
            const long long n2 = n_cols >> 1;
            long long j = lane;
            for (; j + 32 * (kGemvUnroll - 1) < n2; j += 32 * kGemvUnroll) {
                double2 a[kGemvUnroll];
#pragma unroll
                for (int u = 0; u < kGemvUnroll; ++u)
                    a[u] = ldg_stream(row2 + j + 32 * u);
#pragma unroll
                for (int u = 0; u < kGemvUnroll; ++u) {
                    const double2 xv = x2[j + 32 * u];
                    acc[u] = fma(a[u].x, xv.x, acc[u]);
                    acc[u] = fma(a[u].y, xv.y, acc[u]);
                }
            }
            for (; j < n2; j += 32) {
                const double2 a = ldg_stream(row2 + j);
                const double2 xv = x2[j];
                acc[0] = fma(a.x, xv.x, acc[0]);
                acc[0] = fma(a.y, xv.y, acc[0]);
            }
            c = n2 << 1;
            if ((n_cols & 1) && lane == 0)
                acc[1] = fma(row[c], x[c], acc[1]);
        } else {
            for (c = lane; c < n_cols; c += 32)
                acc[0] = fma(__ldg(row + c), x[c], acc[0]);
        }
        double s = 0.0;
#pragma unroll
        for (int u = 0; u < kGemvUnroll; ++u)
            s += acc[u];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
            s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0)
            y[r] = v ? s + v[r] : s;
        r = r_next;
    }
}

struct DenseDev {
    int dev = 0, num_sms = 0;
    Stream stream;
    Event e0, e1, t0, t1;
    long long row_begin[2] = {0, 0}, n_rows[2] = {0, 0};
    DevBuf A[2], x, v, y, ticket, ticket_bg;
};

} // namespace

// the background row streamer of stream_kernels.cuh (design and resource budget there)
namespace skb {

__global__ void __maxnreg__(kStreamMaxNReg) dense_stream_kernel(const StreamArgs a) {
    extern __shared__ __align__(128) unsigned char st_smem[];
    uint64_t *full_bar = reinterpret_cast<uint64_t *>(st_smem + kStreamBarOffset);
    uint64_t *empty_bar = full_bar + kStreamStages;
    int2 *meta = reinterpret_cast<int2 *>(st_smem + kStreamMetaOffset);
    double *red = reinterpret_cast<double *>(st_smem + kStreamRedOffset);
    const int t = threadIdx.x;
    const int n_chunks = (int)((a.n_cols + kStreamCols - 1) / kStreamCols);
    if (t == 0) {
        for (int s = 0; s < kStreamStages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], kStreamConsumers / 32);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (t >= kStreamConsumers) {
        // ---- producer: lanes 0..3 own one row of the group each, lane 4 the segment of x; every lane keeps its own source
        // pointer, so a stage costs one short instruction sequence per lane, not five address computations in one lane
        // (that first version spent ~150 cycles per copy and was bound by it whatever the ring depth) ----
        const int lane = t - kStreamConsumers;
        if (lane > kStreamRows)
            return;
        constexpr unsigned kMask = (2u << kStreamRows) - 1u;
        const long long n_groups = (a.n_rows + kStreamRows - 1) / kStreamRows;
        const uint64_t policy = l2_policy_evict_first();
        long long group = blockIdx.x;
        int s = 0;
        uint32_t empty_parity = 1; // parity of the phase BEFORE the first use: the wait falls through on a fresh barrier
        for (;;) {
            if (group >= n_groups) { // end marker: completes on the arrive alone
                if (lane == 0) {
                    mbar_wait(&empty_bar[s], empty_parity);
                    meta[s] = make_int2(-1, 0);
                    mbar_arrive(&full_bar[s]);
                }
                return;
            }
            // the ticket of the FOLLOWING group is drawn a whole group ahead of its use
            unsigned long long ticket = 0;
            if (lane == 0)
                ticket = atomicAdd(a.next_group, 1ULL);
            const long long row0 = group * kStreamRows;
            const int rows = (int)min((long long)kStreamRows, a.n_rows - row0);
            const double *src = lane < kStreamRows ? a.A + (row0 + lane) * a.n_cols : a.x;
            const bool active = lane == kStreamRows || lane < rows;
            long long left = a.n_cols;
            for (int c = 0; c < n_chunks; ++c) {
                mbar_wait(&empty_bar[s], empty_parity); // the consumers are done with the stage's previous use
                const uint32_t bytes = (uint32_t)(min((long long)kStreamCols, left) * 8);
                unsigned char *dst = st_smem + s * kStreamStageBytes + lane * kStreamRowBytes;
                if (lane == 0) {
                    meta[s] = make_int2((int)group, c);
                    mbar_arrive_expect_tx(&full_bar[s], bytes * (rows + 1));
                }
                if (active) {
                    if (lane < kStreamRows)
                        tma_bulk_g2s_hint(dst, src, bytes, &full_bar[s], policy);
                    else
                        tma_bulk_g2s(dst, src, bytes, &full_bar[s]);
                }
                src += kStreamCols;
                left -= kStreamCols;
                if (++s == kStreamStages) {
                    s = 0;
                    empty_parity ^= 1u;
                }
            }
            group = (long long)gridDim.x + (long long)__shfl_sync(kMask, ticket, 0);
        }
    }

    // ---- consumers ----
    double acc[kStreamRows];
#pragma unroll
    for (int i = 0; i < kStreamRows; ++i)
        acc[i] = 0.0;
    const int n_pairs_last = (int)((a.n_cols - (long long)(n_chunks - 1) * kStreamCols) >> 1); // pairs of the last chunk
    int s = 0;
    uint32_t full_parity = 0;
    for (;; s = (s + 1 == kStreamStages) ? 0 : s + 1, full_parity ^= (s == 0)) {
        mbar_wait(&full_bar[s], full_parity);
        const int2 m = meta[s];
        if (m.x < 0)
            break;
        const int n_pairs = m.y == n_chunks - 1 ? n_pairs_last : kStreamCols / 2;
        const unsigned char *stage = st_smem + s * kStreamStageBytes;
        // thread t owns the column pairs t and 64 + t of the chunk: consecutive lanes read consecutive 16-byte words
#pragma unroll
        for (int h = 0; h < kStreamCols / 2 / kStreamConsumers; ++h) {
            const int p = h * kStreamConsumers + t;
            if (p < n_pairs) {
                const double2 xv = *reinterpret_cast<const double2 *>(stage + kStreamRows * kStreamRowBytes + p * 16);
#pragma unroll
                for (int i = 0; i < kStreamRows; ++i) {
                    // (rows beyond n_rows of the last group hold stale ring data: their sums are never stored)
                    const double2 av = *reinterpret_cast<const double2 *>(stage + i * kStreamRowBytes + p * 16);
                    acc[i] = fma(av.x, xv.x, acc[i]);
                    acc[i] = fma(av.y, xv.y, acc[i]);
                }
            }
        }
        __syncwarp();
        if ((t & 31) == 0)
            mbar_arrive(&empty_bar[s]); // this warp is done with the stage
        if (m.y == n_chunks - 1) { // the group is complete: fixed tree over the 64 consumer threads
#pragma unroll
            for (int i = 0; i < kStreamRows; ++i) {
                double v = acc[i];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1)
                    v += __shfl_xor_sync(0xffffffffu, v, o);
                if ((t & 31) == 0)
                    red[(t >> 5) * kStreamRows + i] = v;
                acc[i] = 0.0;
            }
            asm volatile("bar.sync 1, %0;" ::"n"(kStreamConsumers) : "memory");
            const long long row = (long long)m.x * kStreamRows + t;
            if (t < kStreamRows && row < a.n_rows)
                a.y[row] = red[t] + red[kStreamRows + t];
            asm volatile("bar.sync 1, %0;" ::"n"(kStreamConsumers) : "memory"); // red is free again
        }
    }
}

} // namespace skb

struct skb_dense {
    ~skb_dense() {
        while (!devs.empty()) { // each device's buffers are freed with that device current
            if (devs.back().stream) // (an entry a failed create never reached owns nothing)
                cudaSetDevice(devs.back().dev);
            devs.pop_back();
        }
    }
    std::vector<DenseDev> devs;
    long long rows[2] = {-1, -1}, cols[2] = {0, 0};
    skb_dense_stats stats{};
};

extern "C" {

static int dense_create_impl(const int *ids, int n_gpus, skb_dense **out) {
    if (!out)
        return set_error(SKB_ERR_INVALID, "skb_dense_create: out == NULL");
    *out = nullptr;
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0)
        return set_error(SKB_ERR_NO_DEVICE, "no CUDA device available; this library has no CPU fallback");
    if (n_gpus < 1 || n_gpus > n_dev)
        return set_error(SKB_ERR_INVALID, "skb_dense_create: n_gpus=%d but %d device(s) visible", n_gpus, n_dev);
    std::unique_ptr<skb_dense> dn(new skb_dense);
    dn->devs.resize(n_gpus);
    for (int g = 0; g < n_gpus; ++g) {
        DenseDev &d = dn->devs[g];
        d.dev = ids ? ids[g] : g;
        if (d.dev < 0 || d.dev >= n_dev)
            return set_error(SKB_ERR_INVALID, "skb_dense_create_on: device id %d out of range", d.dev);
        CUDA_TRY(cudaSetDevice(d.dev));
        SKB_TRY(prepare_device(d.dev));
        cudaDeviceProp p;
        CUDA_TRY(cudaGetDeviceProperties(&p, d.dev));
        d.num_sms = p.multiProcessorCount;
        CUDA_TRY(cudaStreamCreateWithFlags(d.stream.out(), cudaStreamNonBlocking));
        CUDA_TRY(cudaEventCreate(d.e0.out()));
        CUDA_TRY(cudaEventCreate(d.e1.out()));
        CUDA_TRY(cudaEventCreate(d.t0.out()));
        CUDA_TRY(cudaEventCreate(d.t1.out()));
    }
    *out = dn.release();
    return SKB_OK;
}

int skb_dense_create(int n_gpus, skb_dense **out) { return dense_create_impl(nullptr, n_gpus, out); }
int skb_dense_create_on(const int *device_ids, int n_gpus, skb_dense **out) {
    if (!device_ids)
        return set_error(SKB_ERR_INVALID, "skb_dense_create_on: device_ids == NULL");
    return dense_create_impl(device_ids, n_gpus, out);
}
int skb_dense_device(const skb_dense *dn, int index, int *device) {
    if (!dn || !device || index < 0 || index >= (int)dn->devs.size())
        return set_error(SKB_ERR_INVALID, "skb_dense_device: bad arguments");
    *device = dn->devs[(size_t)index].dev;
    return SKB_OK;
}

int skb_dense_destroy(skb_dense *dn) {
    if (!dn)
        return SKB_OK;
    for (auto &d : dn->devs)
        if (d.stream)
            cudaStreamSynchronize(d.stream);
    delete dn;
    return SKB_OK;
}

int skb_dense_set_matrix(skb_dense *dn, int op, const double *A, int64_t n_rows, int64_t n_cols) {
    if (!dn || (op != 0 && op != 1) || n_rows < 0 || n_cols < 0 || (n_rows * n_cols > 0 && !A))
        return set_error(SKB_ERR_INVALID, "skb_dense_set_matrix: bad arguments");
    const long long P = (long long)dn->devs.size();
    const long long chunk = (n_rows + P - 1) / P; // contiguous row blocks, periphery.cpp:387-417
    dn->rows[op] = n_rows;
    dn->cols[op] = n_cols;
    for (long long g = 0; g < P; ++g) {
        DenseDev &d = dn->devs[g];
        d.row_begin[op] = std::min<long long>(n_rows, g * chunk);
        d.n_rows[op] = std::min<long long>(n_rows, (g + 1) * chunk) - d.row_begin[op];
        if (d.n_rows[op] == 0 || n_cols == 0)
            continue;
        CUDA_TRY(cudaSetDevice(d.dev));
        SKB_TRY(d.A[op].ensure((size_t)d.n_rows[op] * (size_t)n_cols * 8));
        SKB_TRY(upload_pageable(d.A[op].ptr, A + d.row_begin[op] * n_cols, (size_t)d.n_rows[op] * n_cols * 8, d.stream));
        SKB_TRY(d.ticket_bg.ensure(8));
        SKB_TRY(d.ticket.ensure(8)); // (not at the first apply: no allocation on the matvec path, see skb_flow_group_warmup)
    }
    for (auto &d : dn->devs) {
        CUDA_TRY(cudaSetDevice(d.dev));
        CUDA_TRY(cudaStreamSynchronize(d.stream));
    }
    return SKB_OK;
}

int skb_dense_apply(skb_dense *dn, int op, const double *x, const double *v_add, double *y) {
    if (!dn || (op != 0 && op != 1))
        return set_error(SKB_ERR_INVALID, "skb_dense_apply: bad arguments");
    if (dn->rows[op] < 0)
        return set_error(SKB_ERR_STATE, "skb_dense_apply: skb_dense_set_matrix(op=%d) has not been called", op);
    const long long n_rows = dn->rows[op], n_cols = dn->cols[op];
    if ((n_cols > 0 && !x) || (n_rows > 0 && !y))
        return set_error(SKB_ERR_INVALID, "skb_dense_apply: NULL x or y");
    for (auto &d : dn->devs) {
        if (d.n_rows[op] == 0)
            continue;
        CUDA_TRY(cudaSetDevice(d.dev));
        SKB_TRY(d.x.ensure((size_t)std::max<long long>(n_cols, 1) * 8 + 16));
        SKB_TRY(d.y.ensure((size_t)d.n_rows[op] * 8));
        CUDA_TRY(cudaEventRecord(d.t0, d.stream));
        if (n_cols > 0)
            CUDA_TRY(cudaMemcpyAsync(d.x.ptr, x, (size_t)n_cols * 8, cudaMemcpyHostToDevice, d.stream));
        const double *dv = nullptr;
        if (v_add) {
            SKB_TRY(d.v.ensure((size_t)d.n_rows[op] * 8));
            CUDA_TRY(cudaMemcpyAsync(d.v.ptr, v_add + d.row_begin[op], (size_t)d.n_rows[op] * 8,
                                     cudaMemcpyHostToDevice, d.stream));
            dv = (const double *)d.v.ptr;
        }
        const int vec_ok = (n_cols % 2 == 0) ? 1 : 0; // every row then starts 16-byte aligned
        int occ = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, dense_gemv_kernel, 256, 0) != cudaSuccess || occ < 1)
            occ = 2;
        const int blocks = d.num_sms * occ; // all warps resident; further rows come from the ticket counter
        SKB_TRY(d.ticket.ensure(8));
        CUDA_TRY(cudaMemsetAsync(d.ticket.ptr, 0, 8, d.stream));
        CUDA_TRY(cudaEventRecord(d.e0, d.stream));
        dense_gemv_kernel<<<blocks, 256, 0, d.stream>>>((const double *)d.A[op].ptr, (const double *)d.x.ptr, dv,
                                                        (double *)d.y.ptr, d.n_rows[op], n_cols, vec_ok,
                                                        (unsigned long long *)d.ticket.ptr);
        CUDA_TRY(cudaGetLastError());
        count_launch(1);
        CUDA_TRY(cudaEventRecord(d.e1, d.stream));
        CUDA_TRY(cudaMemcpyAsync(y + d.row_begin[op], d.y.ptr, (size_t)d.n_rows[op] * 8, cudaMemcpyDeviceToHost,
                                 d.stream));
        CUDA_TRY(cudaEventRecord(d.t1, d.stream));
    }
    double k = 0, t = 0;
    for (auto &d : dn->devs) {
        if (d.n_rows[op] == 0)
            continue;
        CUDA_TRY(cudaSetDevice(d.dev));
        CUDA_TRY(cudaStreamSynchronize(d.stream));
        float ms = 0;
        if (cudaEventElapsedTime(&ms, d.e0, d.e1) == cudaSuccess)
            k = std::max(k, (double)ms);
        if (cudaEventElapsedTime(&ms, d.t0, d.t1) == cudaSuccess)
            t = std::max(t, (double)ms);
    }
    dn->stats.kernel_ms = k;
    dn->stats.total_ms = t;
    dn->stats.bytes = 8 * n_rows * n_cols;
    return SKB_OK;
}

int skb_dense_shape(const skb_dense *dn, int op, int64_t *n_rows, int64_t *n_cols) {
    if (!dn || (op != 0 && op != 1) || !n_rows || !n_cols)
        return set_error(SKB_ERR_INVALID, "skb_dense_shape: bad arguments");
    *n_rows = dn->rows[op];
    *n_cols = dn->cols[op];
    return SKB_OK;
}

int skb_dense_apply_device(skb_dense *dn, int op, const double *d_x, const double *d_v_add, double *d_y,
                           void *stream) {
    if (!dn || (op != 0 && op != 1))
        return set_error(SKB_ERR_INVALID, "skb_dense_apply_device: bad arguments");
    if (dn->rows[op] < 0)
        return set_error(SKB_ERR_STATE, "skb_dense_apply_device: skb_dense_set_matrix(op=%d) has not been called", op);
    if (dn->devs.size() != 1)
        return set_error(SKB_ERR_INVALID, "skb_dense_apply_device needs a single-device handle (this one spans %d)",
                         (int)dn->devs.size());
    const long long n_rows = dn->rows[op], n_cols = dn->cols[op];
    if (n_rows == 0)
        return SKB_OK;
    if ((n_cols > 0 && !d_x) || !d_y)
        return set_error(SKB_ERR_INVALID, "skb_dense_apply_device: NULL x or y");
    DenseDev &d = dn->devs[0];
    cudaStream_t st = (cudaStream_t)stream;
    CUDA_TRY(cudaSetDevice(d.dev));
    const int vec_ok = (n_cols % 2 == 0 && ((uintptr_t)d_x & 15) == 0) ? 1 : 0;
    int occ = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, dense_gemv_kernel, 256, 0) != cudaSuccess || occ < 1)
        occ = 2;
    SKB_TRY(d.ticket.ensure(8));
    CUDA_TRY(cudaMemsetAsync(d.ticket.ptr, 0, 8, st));
    dense_gemv_kernel<<<d.num_sms * occ, 256, 0, st>>>((const double *)d.A[op].ptr, d_x, d_v_add, d_y, n_rows, n_cols,
                                                      vec_ok, (unsigned long long *)d.ticket.ptr);
    CUDA_TRY(cudaGetLastError());
    count_launch(1);
    dn->stats.kernel_ms = 0;
    dn->stats.total_ms = 0;
    dn->stats.bytes = 8 * n_rows * n_cols;
    return SKB_OK;
}

int skb_dense_apply_background_device(skb_dense *dn, int op, const double *d_x, double *d_y, void *stream) {
    if (!dn || (op != 0 && op != 1))
        return set_error(SKB_ERR_INVALID, "skb_dense_apply_background_device: bad arguments");
    if (dn->rows[op] < 0)
        return set_error(SKB_ERR_STATE, "skb_dense_apply_background_device: skb_dense_set_matrix(op=%d) has not been "
                                        "called", op);
    if (dn->devs.size() != 1)
        return set_error(SKB_ERR_INVALID, "skb_dense_apply_background_device needs a single-device handle (this one "
                                          "spans %d)", (int)dn->devs.size());
    const long long n_rows = dn->rows[op], n_cols = dn->cols[op];
    if (n_rows == 0)
        return SKB_OK;
    if ((n_cols > 0 && !d_x) || !d_y)
        return set_error(SKB_ERR_INVALID, "skb_dense_apply_background_device: NULL x or y");
    // the TMA streamer needs 16-byte aligned rows and x; anything else takes the classic kernel on the same stream
    if (n_cols % 2 != 0 || ((uintptr_t)d_x & 15) != 0 || n_cols == 0)
        return skb_dense_apply_device(dn, op, d_x, nullptr, d_y, stream);
    DenseDev &d = dn->devs[0];
    cudaStream_t st = (cudaStream_t)stream;
    CUDA_TRY(cudaSetDevice(d.dev));
    SKB_TRY(d.ticket_bg.ensure(8));
    CUDA_TRY(cudaMemsetAsync(d.ticket_bg.ptr, 0, 8, st));
    StreamArgs a;
    a.A = (const double *)d.A[op].ptr;
    a.x = d_x;
    a.y = d_y;
    a.n_rows = n_rows;
    a.n_cols = n_cols;
    a.next_group = (unsigned long long *)d.ticket_bg.ptr;
    const long long n_groups = (n_rows + kStreamRows - 1) / kStreamRows;
    const unsigned grid = (unsigned)std::min<long long>(d.num_sms, n_groups);
    dense_stream_kernel<<<grid, kStreamThreads, kStreamSmemBytes, st>>>(a);
    CUDA_TRY(cudaGetLastError());
    count_launch(1);
    dn->stats.kernel_ms = 0;
    dn->stats.total_ms = 0;
    dn->stats.bytes = 8 * n_rows * n_cols;
    return SKB_OK;
}

int skb_dense_last_stats(const skb_dense *dn, skb_dense_stats *out) {
    if (!dn || !out)
        return set_error(SKB_ERR_INVALID, "skb_dense_last_stats: NULL");
    *out = dn->stats;
    return SKB_OK;
}

} // extern "C"

int skb::load_dense_kernels() {
    cudaFuncAttributes fa;
    CUDA_TRY(cudaFuncGetAttributes(&fa, dense_gemv_kernel));
    return SKB_OK;
}

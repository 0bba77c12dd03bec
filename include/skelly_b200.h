/*
 * skelly_b200.h -- C ABI of the H100-native pair-interaction backend for SkellySim.
 *
 * Drop-in boundary for the reference's direct "GPU" pair evaluator and its STKFMM call sites
 * (all citations relative to the SkellySim tree):
 *
 *   reference interface                                         replaced by
 *   ----------------------------------------------------------  ------------------------------------
 *   kernels::stokeslet_direct_gpu_impl   include/kernels.hpp:17  skb_stokeslet_direct  (+ the same C++ symbol,
 *   kernels::stresslet_direct_gpu_impl   include/kernels.hpp:19  skb_stresslet_direct    exported by the .so)
 *   kernels::GPUEvaluator (declared, never defined)
 *                                        include/kernels.hpp:136-191  skb_ctx_* / skb_set_* / skb_eval
 *   kernels::FMM<Stk3DFMM>::operator()   include/kernels.hpp:78-122   same (positions cached per timestep,
 *                                                                      strengths shipped per matvec)
 *   FiberContainerFiniteDifference::flow src/core/fiber_container_finite_difference.cpp:172-214  skb_flow_* (skelly_b200_flow.h)
 *   Periphery::flow                      src/core/periphery.cpp:55-79                             skb_flow_* (skelly_b200_flow.h)
 *   BodyContainer::flow                  src/core/body_container.cpp:269-477                      skb_flow_* (skelly_b200_flow.h)
 *   System::apply_matvec (flow part)     src/core/system.cpp:284-316                              skb_flow_matvec (skelly_b200_flow.h)
 *
 * Conventions (identical to the reference, SURVEY.md section 8b):
 *   - all coordinates / strengths / velocities FP64, Eigen column-major 3 x n == AoS xyz: r[3*i + k];
 *     stresslet strength is 9 x n: f[9*i + 3*a + b] (a = normal index, b = density index);
 *   - r = x_trg - x_src; pairs with r == 0 contribute exactly 0 (kernels.cu:39,70);
 *   - skb_*_direct and skb_eval results include 1/(8 pi) and EXCLUDE 1/eta (kernels.cu:26,59; the
 *     C++ wrapper divides, kernels.cpp:358,365); outputs are overwritten unless `accumulate` != 0;
 *   - host pointers unless a function name ends in _device; the caller owns its buffers for the
 *     duration of the call; calls are synchronous (results valid on return) unless stated;
 *   - one caller thread per context at a time (the reference calls evaluators from the single
 *     MPI_THREAD_FUNNELED main thread, skelly_sim.cpp:14);
 *   - every function returns 0 (SKB_OK) or a negative-free error code below;
 *     skb_last_error_string() gives the thread's last message.  The reference's CUDA path prints and
 *     exit()s (kernels.cu:8-15); the C++ wrapper in skelly_b200/kernels.hpp throws std::runtime_error,
 *     which SkellySim's main catches (skelly_sim.cpp:57-64).
 *
 * There is no CPU fallback anywhere behind this interface: without a CUDA device every entry point
 * returns SKB_ERR_NO_DEVICE.
 */
#ifndef SKELLY_B200_H
#define SKELLY_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SKB_API __attribute__((visibility("default")))

enum skb_status {
    SKB_OK = 0,
    SKB_ERR_INVALID = 1,   /* bad argument / size / kind */
    SKB_ERR_CUDA = 2,      /* CUDA runtime error (message has the call site) */
    SKB_ERR_NO_DEVICE = 3, /* no usable CUDA device */
    SKB_ERR_STATE = 4,     /* call sequence error (e.g. eval before set_sources) */
    SKB_ERR_NCCL = 5,      /* NCCL could not be loaded / returned an error */
    SKB_ERR_ALLOC = 6      /* host or device allocation failed */
};

/* pair kernels */
enum skb_kernel {
    SKB_STOKESLET = 0, /* single layer, 3 strengths / source   (kernels.cu:57-77) */
    SKB_STRESSLET = 1  /* double layer, 9 strengths / source   (kernels.cu:24-55) */
};

typedef struct skb_ctx skb_ctx;

/* ---- library ------------------------------------------------------------------------------- */
SKB_API const char *skb_version(void);
SKB_API const char *skb_last_error_string(void);
SKB_API int skb_device_count(int *n_devices);

/* ---- stateless reference-shaped entry points -------------------------------------------------
 * Same argument list as kernels::stokeslet_direct_gpu_impl / stresslet_direct_gpu_impl
 * (include/kernels.hpp:17-20, src/core/kernels.cu:180-188): host pointers, `int` counts, output
 * overwritten, scaled by 1/(8 pi), not by 1/eta.  They run on a process-wide context created on
 * first use (device 0), so repeated calls do not re-allocate (the reference mallocs/frees 4 buffers
 * per call, kernels.cu:154-177). */
SKB_API int skb_stokeslet_direct(const double *r_src, const double *f_src, int n_src, const double *r_trg,
                                 double *u_trg, int n_trg);
SKB_API int skb_stresslet_direct(const double *r_src, const double *f_src, int n_src, const double *r_trg,
                                 double *u_trg, int n_trg);

/* ---- evaluator context (what kernels::GPUEvaluator was meant to be) ---------------------------
 * Positions are uploaded when they change (once per timestep); each matvec ships strengths only.
 * n_gpus > 1: ONE process drives n devices (the reference's direct evaluators require a single MPI
 * rank, system.cpp:618-623): targets are block-partitioned across the devices, every device holds
 * all sources, strengths are distributed by one NCCL all-gather per evaluation. */
SKB_API int skb_ctx_create(int n_gpus, skb_ctx **out);
SKB_API int skb_ctx_create_on(const int *device_ids, int n_gpus, skb_ctx **out);
SKB_API int skb_ctx_destroy(skb_ctx *ctx);
SKB_API int skb_ctx_n_gpus(const skb_ctx *ctx, int *n_gpus);

SKB_API int skb_set_targets(skb_ctx *ctx, const double *r_trg, int64_t n_trg);
SKB_API int skb_set_sources(skb_ctx *ctx, int kind, const double *r_src, int64_t n_src);

/* u_trg[3*n_trg] (=|+=) (1/(8 pi)) * sum over the `kind` sources.  f_src: 3 (SL) or 9 (DL) per source. */
SKB_API int skb_eval(skb_ctx *ctx, int kind, const double *f_src, double *u_trg, int accumulate);

/* Both source classes in one call: u = SL(f_sl) + DL(f_dl); either pointer may be NULL (class skipped). */
SKB_API int skb_eval_fused(skb_ctx *ctx, const double *f_sl, const double *f_dl, double *u_trg);

/* Double layer with the strength formed on the device from normals and density,
 * f = 2 eta n (x) rho  (periphery.cpp:68-71, body_container.cpp:296-302), shipping 3 instead of 9
 * doubles per source per matvec.  Normals are cached like positions. */
SKB_API int skb_set_source_normals(skb_ctx *ctx, const double *normals, int64_t n_src);
SKB_API int skb_eval_double_layer(skb_ctx *ctx, const double *density, double eta, double *u_trg, int accumulate);

/* Opt-in fused self-exclusion (SURVEY.md 8f N3; the reference computes all pairs and then subtracts each fiber's own
 * dense block, fiber_container_finite_difference.cpp:203-210, fiber_finite_difference.cpp:56): give every Stokeslet
 * source an id (its fiber index).  The targets must START with the sources (checked); a pair (target i < n_src,
 * source j) with ids[i] == ids[j] then contributes exactly 0 -- decided in the integer pipe next to the r == 0 rule,
 * no FP64 work added.  Differs from compute-then-subtract only where the reference's regularised branch would act
 * (two distinct nodes of one fiber closer than 1e-5, kernels.cpp:176-184) and by the absence of the cancellation
 * rounding.  ids == NULL switches it off; skb_set_sources(SKB_STOKESLET) clears it. */
SKB_API int skb_set_source_exclusion_ids(skb_ctx *ctx, const int32_t *ids, int64_t n_src);

/* ---- device-pointer entry points (single-GPU contexts) ----------------------------------------
 * For hosts that already own device memory and a stream (one rank per GPU under NCCL: the caller
 * all-gathers strengths itself, then evaluates its target block).  Asynchronous on `stream`, a
 * cudaStream_t passed as void* and used verbatim (NULL = CUDA's legacy default stream); the caller
 * synchronises that stream.  skb_sync only waits for the context's own (host-pointer path) stream. */
SKB_API int skb_set_targets_device(skb_ctx *ctx, const double *d_r_trg, int64_t n_trg, void *stream);
SKB_API int skb_set_sources_device(skb_ctx *ctx, int kind, const double *d_r_src, int64_t n_src, void *stream);
SKB_API int skb_eval_device(skb_ctx *ctx, int kind, const double *d_f_src, double *d_u_trg, int accumulate,
                            void *stream);
SKB_API int skb_sync(skb_ctx *ctx);

/* ---- instrumentation -------------------------------------------------------------------------- */
typedef struct skb_eval_stats {
    double kernel_ms;      /* CUDA-event time of the pair kernel(s) of the last evaluation (max over devices) */
    double total_ms;       /* CUDA-event time of the whole device-side evaluation incl. pack / reduce / copies */
    int64_t n_pairs;       /* source x target pairs evaluated */
    int32_t launches;      /* kernels launched by the last evaluation (all devices) */
    int32_t targets_per_thread;
    int32_t source_splits;
    int32_t grid_ctas;
} skb_eval_stats;
SKB_API int skb_last_eval_stats(const skb_ctx *ctx, skb_eval_stats *out);
/* total number of kernels this library has launched in this process */
SKB_API int64_t skb_launch_count(void);
/* total number of times this library's grow-only device buffers have allocated (cudaMalloc) in this process: a call
 * documented to allocate nothing leaves it unchanged */
SKB_API int64_t skb_buffer_alloc_count(void);
/* tuning overrides (0 = automatic): targets per thread in {1,2,4,8}, source splits >= 1 */
SKB_API int skb_ctx_set_tuning(skb_ctx *ctx, int targets_per_thread, int source_splits);

/* Stokeslet self-interaction with Newton's third law: when the sources are bit-identical to the leading targets
 * (the fiber -> fiber block of System::apply_matvec, system.cpp:284-299) each pair's geometry is evaluated once
 * for both directions.  mode: -1 automatic (default: on for >= 4096 such sources on single-GPU contexts),
 * 0 never, 1 whenever applicable.  Results stay within the same 1e-12 gate; summation order differs from the
 * plain kernel, and stays bitwise reproducible run to run. */
SKB_API int skb_ctx_set_symmetric(skb_ctx *ctx, int mode);
/* One rank per GPU with the symmetric kernel: this context evaluates only the block rows of the self-interaction
 * owned by `part` (of `n_parts`, serpentine over rows).  The leading n_src rows of the result are then PARTIAL sums:
 * the caller adds the parts (one all-reduce of 24 B x n_src per evaluation); rows beyond n_src are complete.  With
 * n_parts == 1 (default) nothing changes.  Only takes effect when the symmetric kernel is used. */
SKB_API int skb_ctx_set_sym_partition(skb_ctx *ctx, int part, int n_parts);
/* 1 if the last Stokeslet evaluation of this context went through the symmetric kernel, else 0 */
SKB_API int skb_ctx_last_eval_was_symmetric(const skb_ctx *ctx, int *yes);

/* duration (CUDA events on the launch stream, valid once that stream has passed them) and ordered-pair count of the
 * last launch of the symmetric kernel on the context's first device; 0 / 0 when it has not run */
SKB_API int skb_ctx_last_sym_kernel(const skb_ctx *ctx, double *ms, int64_t *pairs);

/* ---- host-side planners, callable without a GPU (unit-tested on CPU) ------------------------------------------
 * Launch plan of the plain pair kernel for a problem of n_src sources x n_trg targets on a device with `num_sms`
 * SMs and the given resident-CTA counts for T = 1, 2, 4, 8 targets per thread. */
SKB_API int skb_plan_query(int kind, int64_t n_trg, int64_t n_src, int num_sms, const int *occupancy4, int force_T,
                           int force_S, int *T, int *n_splits, int *tiles_per_split, int *grid_x);
/* Work items of the symmetric kernel for `n_blocks` node blocks and the rows owned by `part` of `n_parts`:
 * items4[4*i..] = (I, g0, g1, slot) in launch order (at most max_items are written): block I meets the 32-node groups
 * [g0, g1), all of them beyond block I (a block is skb_sym_groups_per_block() groups); row_begin[n_blocks + 1]. */
SKB_API int skb_sym_plan_query(int n_blocks, int part, int n_parts, int num_sms, int max_items, int *items4,
                               int *n_items, int *row_begin);
SKB_API int skb_sym_groups_per_block(void);

/* Pure DFMA micro-benchmark on the context's first device: returns achieved FP64 FMA/s * 2 (flop/s).
 * SURVEY.md section 8d asks for the measured FP64 roofline denominator next to the datasheet value. */
SKB_API int skb_measure_fp64_peak(skb_ctx *ctx, double *flops_per_s);

#ifdef __cplusplus
}
#endif
#endif /* SKELLY_B200_H */

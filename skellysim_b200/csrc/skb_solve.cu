// skb_solve.cu -- Solver::solve (solver_hydro.cpp:64-95) on the device: right-preconditioned restarted GMRES over the
// whole-system operator and preconditioner of a flow (include/skelly_b200_flow.h, skb_flow_solve_system).  The vector
// passes are krylov_kernels.cuh; the Hessenberg scalars, the Givens rotations and every decision are on the host.
#include "krylov_kernels.cuh"
#include "skb_flow.hpp"

#include <algorithm>
#include <cmath>
#include <cstring>

using namespace skb;

namespace {
constexpr int kCtasPerSm = 4;                  // of the row-block passes: fixed per device, so is every sum's order
constexpr double kBreakdown = 16.0 * 0x1p-53;  // a new vector at most this fraction of its norm before ICGS: breakdown
constexpr int kWords = 4;                      // nrm[0] = |w|^2 after pass C, nrm[1] = |r|^2 of the last residual

unsigned elementwise_grid(long long n) { return (unsigned)std::clamp<long long>((n + 255) / 256, 1, 4096); }
} // namespace

// device words of small_ and host_: h1 [ldp] | h2 [ldp] | nrm [kWords] | y [ldp]
int Krylov::setup(long long n, int num_blocks, int num_sms, const std::array<long long, 6> &key) {
    const long long ld = (n + 31) / 32 * 32;
    const long long want = std::max<long long>(1, (n + 31) / 32); // at least one tile per CTA
    const long long ctas0 = std::min<long long>((long long)kCtasPerSm * num_sms, want);
    const long long rows_per = std::max<long long>(32, ((n + ctas0 - 1) / ctas0 + 31) / 32 * 32);
    const int ctas = (int)std::max<long long>(1, (n + rows_per - 1) / rows_per); // n = 0: one CTA writing zeros
    const int ldp = num_blocks + 2;
    set_ = false; // a failed allocation leaves no workspace
    SKB_TRY(V_.ensure((size_t)ld * (num_blocks + 1) * 8 + 8));
    SKB_TRY(z_.ensure((size_t)n * 8 + 8));
    SKB_TRY(u_.ensure((size_t)n * 8 + 8));
    SKB_TRY(b_.ensure((size_t)n * 8 + 8));
    SKB_TRY(x_.ensure((size_t)n * 8 + 8));
    SKB_TRY(part_.ensure((size_t)ctas * ldp * 8));
    SKB_TRY(small_.ensure((size_t)(3 * ldp + kWords) * 8));
    host_.reset();
    CUDA_TRY(cudaMallocHost((void **)host_.out(), (size_t)(3 * ldp + kWords) * 8));
    if (!done_.get())
        CUDA_TRY(cudaEventCreateWithFlags(done_.out(), cudaEventDisableTiming));
    // loaded now: a group member must not load a kernel lazily while a peer on the same device spins on a flag
    cudaFuncAttributes fa;
    CUDA_TRY(cudaFuncGetAttributes(&fa, krylov_pass_kernel<kDots>));
    CUDA_TRY(cudaFuncGetAttributes(&fa, krylov_pass_kernel<kUpdateDots>));
    CUDA_TRY(cudaFuncGetAttributes(&fa, krylov_pass_kernel<kUpdateNorm>));
    CUDA_TRY(cudaFuncGetAttributes(&fa, krylov_combine_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, krylov_residual_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, krylov_scale_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, krylov_gemv_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, krylov_axpy_kernel));
    H_.assign((size_t)(num_blocks + 1) * num_blocks, 0.0);
    cs_.assign(num_blocks, 0.0);
    sn_.assign(num_blocks, 0.0);
    g_.assign(num_blocks + 1, 0.0);
    y_.assign(num_blocks, 0.0);
    n_ = n;
    ld_ = ld;
    rows_per_ = rows_per;
    ctas_ = ctas;
    ldp_ = ldp;
    m_cap_ = num_blocks;
    key_ = key;
    set_ = true;
    return SKB_OK;
}

// one pass over the k columns of V and the vector d_w, then the fixed-order combine of its CTA partials into d_out
int Krylov::pass(int which, int k, double *d_w, const double *d_coef, double *d_out, const Reduce &reduce,
                 cudaStream_t st, int *launches) {
    const double *V = (const double *)V_.ptr;
    double *part = (double *)part_.ptr;
    const size_t smem = (size_t)(2 * k + 1 + 32 + 32 * kKrylovWarps) * 8;
    int m = 1;
    if (which == kDots) {
        krylov_pass_kernel<kDots><<<ctas_, kKrylovThreads, smem, st>>>(V, ld_, k, d_w, d_coef, n_, rows_per_, part,
                                                                       ldp_);
        m = k + 1;
    } else if (which == kUpdateDots) {
        krylov_pass_kernel<kUpdateDots><<<ctas_, kKrylovThreads, smem, st>>>(V, ld_, k, d_w, d_coef, n_, rows_per_,
                                                                             part, ldp_);
        m = k;
    } else {
        krylov_pass_kernel<kUpdateNorm><<<ctas_, kKrylovThreads, smem, st>>>(V, ld_, k, d_w, d_coef, n_, rows_per_,
                                                                             part, ldp_);
    }
    krylov_combine_kernel<<<m, kCombineThreads, 0, st>>>(part, ctas_, ldp_, d_out);
    SKB_TRY(launched(launches, 2));
    return reduce ? reduce(d_out, m) : SKB_OK;
}

int Krylov::residual(const double *d_b, const double *d_ax, const Reduce &reduce, cudaStream_t st, int *launches) {
    double *nrm = (double *)small_.ptr + 2 * ldp_;
    krylov_residual_kernel<<<ctas_, kKrylovThreads, 0, st>>>(d_b, d_ax, (double *)V_.ptr, n_, rows_per_,
                                                             (double *)part_.ptr, ldp_);
    krylov_combine_kernel<<<1, kCombineThreads, 0, st>>>((const double *)part_.ptr, ctas_, ldp_, nrm + 1);
    SKB_TRY(launched(launches, 2));
    return reduce ? reduce(nrm + 1, 1) : SKB_OK;
}

int Krylov::wait(cudaStream_t st) {
    CUDA_TRY(cudaMemcpyAsync(host_.get(), small_.ptr, (size_t)(2 * ldp_ + kWords) * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaEventRecord(done_, st));
    CUDA_TRY(cudaEventSynchronize(done_));
    return SKB_OK;
}

int Krylov::solve(const Apply &A, const Apply &P_inv, const Reduce &reduce, const double *d_b, double *d_x, double tol,
                  int num_blocks, int max_iters, cudaStream_t st, skb_solve_info *info, double *history,
                  int *launches) {
    const long long n = n_, ld = ld_;
    const int m = num_blocks;
    double *V = (double *)V_.ptr, *z = (double *)z_.ptr, *u = (double *)u_.ptr;
    double *d_h1 = (double *)small_.ptr, *d_h2 = d_h1 + ldp_, *d_nrm = d_h2 + ldp_, *d_y = d_nrm + kWords;
    const double *h1 = host_.get(), *h2 = h1 + ldp_, *nrm = h2 + ldp_;
    double *h_y = host_.get() + 2 * ldp_ + kWords;
    std::memset(info, 0, sizeof(*info));

    CUDA_TRY(cudaMemsetAsync(d_x, 0, (size_t)n * 8, st));
    SKB_TRY(residual(d_b, nullptr, reduce, st, launches)); // r0 = b into V col 0
    SKB_TRY(wait(st));
    const double bnorm = std::sqrt(nrm[1]);
    const double target = tol * bnorm;
    if (history)
        history[0] = bnorm > 0 ? 1.0 : 0.0;
    double beta = bnorm, est = bnorm; // the explicit residual norm at the cycle's start; the implicit estimate
    int total = 0;
    bool converged = beta <= target;  // ||b|| = 0 (or tol >= 1): x0 = 0 is the answer
    while (!converged && total < max_iters) {
        // v_0 = r / ||r||
        krylov_scale_kernel<<<elementwise_grid(n), 256, 0, st>>>(V, n, d_nrm + 1);
        SKB_TRY(launched(launches));
        std::fill(g_.begin(), g_.end(), 0.0);
        g_[0] = beta;
        int k = 0;
        while (k < m && total < max_iters) {
            double *v = V + (long long)k * ld, *w = V + (long long)(k + 1) * ld;
            SKB_TRY(P_inv(v, z)); // z = P^-1 v_k, w = A z
            SKB_TRY(A(z, w));
            SKB_TRY(pass(kDots, k + 1, w, nullptr, d_h1, reduce, st, launches));
            SKB_TRY(pass(kUpdateDots, k + 1, w, d_h1, d_h2, reduce, st, launches));
            SKB_TRY(pass(kUpdateNorm, k + 1, w, d_h2, d_nrm, reduce, st, launches));
            SKB_TRY(wait(st));
            double *h = &H_[(size_t)k * (m + 1)];
            for (int i = 0; i <= k; ++i)
                h[i] = h1[i] + h2[i];
            const double w0 = std::sqrt(h1[k + 1]);
            double bet = std::sqrt(nrm[0]);
            const bool breakdown = !(bet > kBreakdown * w0); // 0, or rounding of an exactly invariant space
            if (breakdown)
                bet = 0.0;
            h[k + 1] = bet;
            for (int i = 0; i < k; ++i) { // the earlier rotations, then the one that zeroes h[k + 1]
                const double t = cs_[i] * h[i] + sn_[i] * h[i + 1];
                h[i + 1] = -sn_[i] * h[i] + cs_[i] * h[i + 1];
                h[i] = t;
            }
            const double r = std::hypot(h[k], h[k + 1]);
            cs_[k] = r > 0 ? h[k] / r : 1.0;
            sn_[k] = r > 0 ? h[k + 1] / r : 0.0;
            h[k] = r;
            h[k + 1] = 0.0;
            g_[k + 1] = -sn_[k] * g_[k];
            g_[k] = cs_[k] * g_[k];
            ++k;
            ++total;
            est = std::fabs(g_[k]);
            if (history)
                history[total] = est / bnorm;
            if (breakdown || est <= target)
                break;
            krylov_scale_kernel<<<elementwise_grid(n), 256, 0, st>>>(w, n, d_nrm);
            SKB_TRY(launched(launches));
        }
        // y = R^-1 g over the leading columns with a non-zero diagonal; x += P^-1 V y
        int kk = 0;
        while (kk < k && H_[(size_t)kk * (m + 1) + kk] != 0.0)
            ++kk;
        for (int i = kk - 1; i >= 0; --i) {
            double s = g_[i];
            for (int j = i + 1; j < kk; ++j)
                s -= H_[(size_t)j * (m + 1) + i] * y_[j];
            y_[i] = s / H_[(size_t)i * (m + 1) + i];
        }
        if (kk > 0) {
            std::memcpy(h_y, y_.data(), (size_t)kk * 8);
            CUDA_TRY(cudaMemcpyAsync(d_y, h_y, (size_t)kk * 8, cudaMemcpyHostToDevice, st));
            krylov_gemv_kernel<<<elementwise_grid(n), kKrylovThreads, (size_t)kk * 8, st>>>(V, ld, kk, d_y, u, n);
            SKB_TRY(launched(launches));
            SKB_TRY(P_inv(u, z));
            krylov_axpy_kernel<<<elementwise_grid(n), 256, 0, st>>>(d_x, z, n);
            SKB_TRY(launched(launches));
        }
        // the explicit residual r = b - A x, into V col 0 for a restart
        SKB_TRY(A(d_x, u));
        SKB_TRY(residual(d_b, u, reduce, st, launches));
        SKB_TRY(wait(st));
        beta = std::sqrt(nrm[1]);
        converged = beta <= target;
        if (!converged && total < max_iters)
            ++info->restarts;
    }
    info->converged = converged;
    info->iterations = total;
    info->implicit_residual = bnorm > 0 ? est / bnorm : 0.0;
    info->explicit_residual = bnorm > 0 ? beta / bnorm : 0.0;
    info->residual = beta;
    return SKB_OK;
}

int skb::solve_scalar_args(const char *who, double tol, int num_blocks, int max_iters) {
    if (!(tol > 0) || !std::isfinite(tol))
        return set_error(SKB_ERR_INVALID, "%s: tol = %g (must be finite and > 0)", who, tol);
    if (num_blocks < 1 || num_blocks > kMaxKrylov)
        return set_error(SKB_ERR_INVALID, "%s: num_blocks = %d (must be in [1, %d])", who, num_blocks, kMaxKrylov);
    if (max_iters < 0)
        return set_error(SKB_ERR_INVALID, "%s: max_iters = %d", who, max_iters);
    return SKB_OK;
}

// the refusals of the two system calls the solve makes (a group member's local-vector calls, else the single-device
// ones): dn_spc holds stresslet_plus_complementary, dn_minv M_inv; *n = the (local) solution size, *key its ranges
static int flow_solve_args(skb_flow *fl, skb_dense *dn_spc, skb_dense *dn_minv, const char *who, long long *n,
                           std::array<long long, 6> *key) {
    if (fl->grp.member()) {
        SKB_TRY(group_system_args(fl, dn_spc, who, false));
        SKB_TRY(group_system_args(fl, dn_minv, who, true));
        *n = group_local_size(fl);
        *key = group_ranges(fl);
        return SKB_OK;
    }
    SKB_TRY(system_args(fl, dn_spc, who, false, true));
    SKB_TRY(system_args(fl, dn_minv, who, true, true));
    *n = solution_size(fl);
    *key = {};
    return SKB_OK;
}

// the refusals of every form, before any launch; *n = the (local) solution size, 0 with an empty system: nothing to
// do (info filled).  group: the local-vector call of a group member (dn_spc / dn_minv its rows of the two operators)
static int solve_args(skb_flow *fl, skb_dense *dn_spc, skb_dense *dn_minv, const char *who, bool group, double eta,
                      double tol, int num_blocks, int max_iters, bool args, skb_solve_info *info, long long *n) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (!group && fl->grp.member())
        return set_error(SKB_ERR_INVALID, "%s: a group member solves its local rows with "
                                          "skb_flow_group_solve_system_device", who);
    std::array<long long, 6> key;
    SKB_TRY(flow_solve_args(fl, dn_spc, dn_minv, who, n, &key));
    if (!(eta > 0))
        return set_error(SKB_ERR_INVALID, "%s: eta = %g", who, eta);
    SKB_TRY(solve_scalar_args(who, tol, num_blocks, max_iters));
    if (!info)
        return set_error(SKB_ERR_INVALID, "%s: NULL info", who);
    if (solution_size(fl) == 0) { // every member of an empty system returns here alike
        std::memset(info, 0, sizeof(*info));
        info->converged = 1;
        *n = 0;
        return SKB_OK;
    }
    const Krylov &kry = fl->kry;
    if (!kry.sized_for(*n, key))
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_gmres for the current solution size (%lld) and target "
                                          "ranges", who, *n);
    if (num_blocks > kry.blocks())
        return set_error(SKB_ERR_INVALID, "%s: num_blocks = %d, skb_flow_set_gmres sized the workspace for %d", who,
                         num_blocks, kry.blocks());
    if (!args && *n > 0)
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    if (*n == 0) // a member that owns no row: it still takes part in every exchange
        *n = -1;
    return SKB_OK;
}

// A and P^-1 are the local-vector calls (the single-device calls on a flow that is no member); every launch, theirs and
// the solve's, is counted into the flow's stats
static int run(skb_flow *fl, skb_dense *dn_spc, skb_dense *dn_minv, const double *d_b, double eta, double tol,
               int num_blocks, int max_iters, double *d_x, skb_solve_info *info, double *history, cudaStream_t st) {
    int launches = 0;
    const Krylov::Apply A = [&](const double *in, double *out) -> int {
        SKB_TRY(skb_flow_group_apply_system_matvec_device(fl, dn_spc, in, eta, out, st));
        launches += fl->launches;
        return SKB_OK;
    };
    const Krylov::Apply P_inv = [&](const double *in, double *out) -> int {
        SKB_TRY(skb_flow_group_apply_system_preconditioner_device(fl, dn_minv, in, out, st));
        launches += fl->launches;
        return SKB_OK;
    };
    Group &G = fl->grp;
    Krylov::Reduce reduce;
    if (G.member())
        reduce = [&](double *d_v, int m) -> int { return G.reduce_dots(d_v, m, st, &launches); };
    SKB_TRY(fl->kry.solve(A, P_inv, reduce, d_b, d_x, tol, num_blocks, max_iters, st, info, history, &launches));
    fl->pairs = 0;
    fl->launches = launches;
    return device_stats(fl);
}

// a group member (skb_flow_set_gmres): the fiber build's and the links' buffers for its own fibers at their final size
// (FiberOps::size_build, BodyOps::size_links); else nothing
static int flow_size_group_step(skb_flow *fl) {
    if (!fl->grp.member())
        return SKB_OK;
    CUDA_TRY(cudaSetDevice(fl->dev));
    OwnFibers own;
    SKB_TRY(own_fibers(fl, "skb_flow_set_gmres", own));
    SKB_TRY(fl->ops.size_build(own));
    return fl->bodies.size_links(own.count(), fl->n_bodies);
}

extern "C" {

int skb_flow_set_gmres(skb_flow *fl, int num_blocks) {
    const char *who = "skb_flow_set_gmres";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (num_blocks < 1 || num_blocks > kMaxKrylov)
        return set_error(SKB_ERR_INVALID, "%s: num_blocks = %d (must be in [1, %d])", who, num_blocks, kMaxKrylov);
    long long n = 0;
    std::array<long long, 6> key;
    SKB_TRY(flow_gmres_size(fl, who, &n, &key));
    SKB_TRY(fl->kry.setup(n, num_blocks, fl->fib[1].info.num_sms, key));
    // the buffers of skb_flow_step / skb_mflow_step / skb_flow_group_step_device beside the solve's
    SKB_TRY(fl->stepbuf.size(fl->n_fibers, fl->n_fib, fl->n_bodies));
    SKB_TRY(fl->shape.size(fl->n_fib));
    return flow_size_group_step(fl);
}

int skb_flow_solve_system(skb_flow *fl, skb_dense *dn, const double *rhs, double eta, double tol, int num_blocks,
                          int max_iters, double *x, skb_solve_info *info, double *history) {
    long long n = 0;
    SKB_TRY(solve_args(fl, dn, dn, "skb_flow_solve_system", false, eta, tol, num_blocks, max_iters, rhs && x, info,
                       &n));
    if (n == 0)
        return SKB_OK;
    const Krylov &kry = fl->kry;
    const cudaStream_t st = fl->stream;
    CUDA_TRY(cudaMemcpyAsync(kry.stage_b(), rhs, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    SKB_TRY(run(fl, dn, dn, kry.stage_b(), eta, tol, num_blocks, max_iters, kry.stage_x(), info, history, st));
    CUDA_TRY(cudaMemcpyAsync(x, kry.stage_x(), (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return SKB_OK;
}

int skb_flow_solve_system_device(skb_flow *fl, skb_dense *dn, const double *d_rhs, double eta, double tol,
                                 int num_blocks, int max_iters, double *d_x, skb_solve_info *info, double *history,
                                 void *stream) {
    long long n = 0;
    SKB_TRY(solve_args(fl, dn, dn, "skb_flow_solve_system_device", false, eta, tol, num_blocks, max_iters,
                       d_rhs && d_x, info, &n));
    if (n == 0)
        return SKB_OK;
    return run(fl, dn, dn, d_rhs, eta, tol, num_blocks, max_iters, d_x, info, history, (cudaStream_t)stream);
}

int skb_flow_group_solve_system_device(skb_flow *fl, skb_dense *dn_spc, skb_dense *dn_minv, const double *d_rhs_local,
                                       double eta, double tol, int num_blocks, int max_iters, double *d_x_local,
                                       skb_solve_info *info, double *history, void *stream) {
    long long n = 0;
    SKB_TRY(solve_args(fl, dn_spc, dn_minv, "skb_flow_group_solve_system_device", true, eta, tol, num_blocks,
                       max_iters, d_rhs_local && d_x_local, info, &n));
    if (n == 0)
        return SKB_OK;
    const bool none = n < 0; // owns no row: the workspace's own buffers stand in for the empty vectors
    const Krylov &kry = fl->kry;
    return run(fl, dn_spc, dn_minv, none ? kry.stage_b() : d_rhs_local, eta, tol, num_blocks, max_iters,
               none ? kry.stage_x() : d_x_local, info, history, (cudaStream_t)stream);
}

} // extern "C"

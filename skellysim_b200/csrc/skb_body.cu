// skb_body.cu -- the bodies' per-timestep operators and the fiber-body links of a flow (BodyOps, skb_internal.hpp): their
// checks and uploads, and the launches of body_ops.cuh and of the body preconditioner's GEMV.  Knows nothing of skb_flow:
// skb_matvec.cu hands it the geometry, the fibers and their operators.
#include "body_ops.cuh"
#include "fiber_ops.cuh"
#include "skb_internal.hpp"

#include <algorithm>
#include <climits>
#include <cmath>
#include <vector>

using namespace skb;

static int launched(int *launches) {
    CUDA_TRY(cudaGetLastError());
    count_launch(1);
    *launches += 1;
    return SKB_OK;
}

static int put(DevBuf &b, const void *h, size_t bytes, cudaStream_t st) {
    if (bytes == 0)
        return SKB_OK;
    SKB_TRY(b.ensure(bytes));
    CUDA_TRY(cudaMemcpyAsync(b.ptr, h, bytes, cudaMemcpyHostToDevice, st));
    return SKB_OK;
}

int BodyOps::set_operators(const int *n_nodes, int n_bodies, long long n_body_nodes, const double *r_body,
                           const double *centers, const double *node_weights, const double *ex, const double *ey,
                           const double *ez, const double *A_inv, cudaStream_t st, long long lo, long long hi) {
    const char *who = "skb_flow_set_body_operators";
    const bool windowed = hi >= 0;
    std::vector<BodyItem> items((size_t)n_bodies);
    std::vector<FiberGemvItem> gemv;
    long long nodes = 0, sol = 0, inv = 0;
    long long inv_first = 0, inv_own = 0; // windowed: the owned bodies' inverses, contiguous in A_inv
    int max_cols = 0, b0 = n_bodies, b1 = 0;
    for (int b = 0; b < n_bodies; ++b) {
        const int n = n_nodes[b];
        if (n < 1)
            return set_error(SKB_ERR_INVALID, "%s: body %d has %d nodes", who, b, n);
        items[(size_t)b] = BodyItem{nodes, sol, n, 0};
        const int m = 3 * n + 6;
        if (!windowed) {
            for (int r0 = 0; r0 < m; r0 += kFiberGemvRows)
                gemv.push_back(FiberGemvItem{inv, sol, sol, m, m, r0, n, b, 0});
        } else if (nodes < hi && nodes + n > lo) {
            // the owned rows of this body: node rows [r_lo, r_hi), and [3n, 3n + 6) if its first node is owned; a
            // 32-row block that reaches any of them is evaluated (the other rows of the block are never read)
            if (b0 > b)
                b0 = b, inv_first = inv;
            b1 = b + 1;
            const int r_lo = 3 * (int)(std::max(lo, nodes) - nodes), r_hi = 3 * (int)(std::min(hi, nodes + n) - nodes);
            const bool six = nodes >= lo;
            for (int r0 = 0; r0 < m; r0 += kFiberGemvRows) {
                const int r1 = r0 + kFiberGemvRows;
                if ((r0 < r_hi && r1 > r_lo) || (six && r1 > 3 * n))
                    gemv.push_back(FiberGemvItem{inv - inv_first, sol, sol, m, m, r0, n, b, 0});
            }
            inv_own = inv + (long long)m * m - inv_first;
        }
        max_cols = std::max(max_cols, m);
        nodes += n;
        sol += m;
        inv += (long long)m * m;
    }
    if (!windowed)
        inv_own = inv;
    if (nodes != n_body_nodes)
        return set_error(SKB_ERR_INVALID, "%s: the bodies' node counts sum to %lld, skb_flow_set_bodies has %lld nodes",
                         who, nodes, n_body_nodes);
    for (long long i = 0; i < nodes; ++i)
        if (!(node_weights[i] > 0))
            return set_error(SKB_ERR_INVALID, "%s: node_weights[%lld] = %g (must be > 0)", who, i, node_weights[i]);
    // fiber_gemv_kernel<0>: x (cols, rounded up to even) and the slice partials
    const size_t smem = ((size_t)((max_cols + 1) & ~1) + kFiberGemvThreads) * sizeof(double);
    if (A_inv && smem > kFiberGemvSmemMax)
        return set_error(SKB_ERR_INVALID, "%s: a body of %d unknowns exceeds the shared memory of the preconditioner's "
                                          "GEMV", who, max_cols);
    ops_set_ = inv_set_ = false;
    SKB_TRY(put(items_, items.data(), items.size() * sizeof(BodyItem), st));
    SKB_TRY(put(r_, r_body, (size_t)nodes * 24, st));
    SKB_TRY(put(centers_, centers, (size_t)n_bodies * 24, st));
    SKB_TRY(put(weights_, node_weights, (size_t)nodes * 8, st));
    SKB_TRY(put(ex_, ex, (size_t)nodes * 24, st));
    SKB_TRY(put(ey_, ey, (size_t)nodes * 24, st));
    SKB_TRY(put(ez_, ez, (size_t)nodes * 24, st));
    SKB_TRY(put(gemv_items_, gemv.data(), gemv.size() * sizeof(FiberGemvItem), st));
    SKB_TRY(dens_.ensure((size_t)nodes * 24 + 8));
    SKB_TRY(force_.ensure((size_t)n_bodies * 24 + 8));
    SKB_TRY(torque_.ensure((size_t)n_bodies * 24 + 8));
    if (A_inv && inv_own > 0) {
        SKB_TRY(a_inv_.ensure((size_t)inv_own * 8));
        SKB_TRY(upload_pageable(a_inv_.ptr, A_inv + inv_first, (size_t)inv_own * 8, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st)); // the host tables above go out of scope
    if (windowed) { // a group member's kernels are loaded now: a lazy load at the first launch would wait behind a
                    // peer on the same device spinning on a flag
        cudaFuncAttributes fa;
        CUDA_TRY(cudaFuncGetAttributes(&fa, fiber_link_kernel));
        CUDA_TRY(cudaFuncGetAttributes(&fa, body_sum_kernel));
        CUDA_TRY(cudaFuncGetAttributes(&fa, body_matvec_kernel<true>));
    }
    n_bodies_ = n_bodies;
    sol_size_ = sol;
    windowed_ = windowed;
    win_b0_ = std::min(b0, b1);
    win_b1_ = b1;
    win_lo_ = lo;
    win_hi_ = hi;
    n_gemv_ = (int)gemv.size();
    gemv_smem_ = smem;
    inv_set_ = A_inv != nullptr || n_bodies == 0;
    ops_set_ = true;
    return SKB_OK;
}

int BodyOps::set_links(const OwnFibers &own, const FiberOps &ops, int n_bodies, const double *centers,
                       const int *body, const double *site, const double *rigidity, cudaStream_t st,
                       bool check_only) {
    const char *who = "skb_flow_set_fiber_links";
    const int nfib = own.count();
    std::vector<LinkFiber> lf((size_t)nfib);
    std::vector<int> count((size_t)n_bodies + 1, 0), csr_fib;
    bool any = false;
    for (int f = 0; f < nfib; ++f) {
        const int b = body ? body[f] : -1;
        LinkFiber &l = lf[(size_t)f];
        l = LinkFiber{{0.0, 0.0, 0.0}, 0.0, own.off[own.f0 + f] - own.off[own.f0], 0, own.n[own.f0 + f], b};
        if (b < -1 || b >= n_bodies)
            return set_error(SKB_ERR_INVALID, "%s: fiber %d is bound to body %d (the flow has %d bodies; -1 = free)",
                             who, own.f0 + f, b, n_bodies);
        if (b < 0)
            continue;
        SKB_TRY(ops.derivative_offset(own.f0 + f, l.n_nodes, &l.d2_off)); // the link needs D_2_0 and D_3_0
        for (int k = 0; k < 3; ++k) // get_nucleation_site(i_body, i_site) - body->get_position()  (:209)
            l.s[k] = site[3 * (size_t)f + k] - centers[3 * (size_t)b + k];
        if (l.s[0] * l.s[0] + l.s[1] * l.s[1] + l.s[2] * l.s[2] == 0.0)
            return set_error(SKB_ERR_INVALID, "%s: fiber %d's nucleation site is the centre of body %d (the rotational "
                                              "link condition divides by their distance)", who, own.f0 + f, b);
        l.rigidity = rigidity[f];
        count[(size_t)b + 1]++;
        any = true;
    }
    if (check_only)
        return SKB_OK;
    // bound fibers per body, in container order
    for (int b = 0; b < n_bodies; ++b)
        count[(size_t)b + 1] += count[(size_t)b];
    std::vector<int> fill(count.begin(), count.end() - 1);
    csr_fib.resize((size_t)count[(size_t)n_bodies]);
    for (int f = 0; f < nfib; ++f)
        if (lf[(size_t)f].body >= 0)
            csr_fib[(size_t)fill[(size_t)lf[(size_t)f].body]++] = f;
    links_set_ = false;
    if (any) {
        SKB_TRY(put(link_fibers_, lf.data(), lf.size() * sizeof(LinkFiber), st));
        SKB_TRY(put(csr_begin_, count.data(), count.size() * sizeof(int), st));
        SKB_TRY(put(csr_fib_, csr_fib.data(), csr_fib.size() * sizeof(int), st));
        SKB_TRY(link_.ensure((size_t)nfib * 56));
        SKB_TRY(contrib_.ensure((size_t)nfib * 48));
        CUDA_TRY(cudaStreamSynchronize(st)); // the host tables above go out of scope
    }
    n_fibers_ = nfib;
    any_bound_ = any;
    links_set_ = true;
    return SKB_OK;
}

int BodyOps::links(const FiberOps &ops, const double *d_length, const double *d_x_fib, const double *d_x_bodies,
                   const double **d_link, cudaStream_t st, int *launches) {
    *d_link = nullptr;
    if (n_bodies_ == 0)
        return SKB_OK;
    const bool bound = links_set_ && any_bound_;
    if (bound) {
        const unsigned grid = (unsigned)((n_fibers_ + kLinkWarps - 1) / kLinkWarps);
        fiber_link_kernel<<<grid, 32 * kLinkWarps, 0, st>>>(
            (const LinkFiber *)link_fibers_.ptr, n_fibers_, (const BodyItem *)items_.ptr, ops.class_table(),
            ops.tangents(), d_length, d_x_fib, d_x_bodies, (double *)link_.ptr, (double *)contrib_.ptr);
        SKB_TRY(launched(launches));
        *d_link = (const double *)link_.ptr;
    }
    body_sum_kernel<<<(unsigned)n_bodies_, kBodyThreads, 0, st>>>(
        (const BodyItem *)items_.ptr, bound ? (const int *)csr_begin_.ptr : nullptr, (const int *)csr_fib_.ptr,
        (const double *)contrib_.ptr, d_x_bodies, (double *)dens_.ptr, (double *)force_.ptr, (double *)torque_.ptr);
    return launched(launches);
}

int BodyOps::matvec(const double *d_x_bodies, const double *d_v_bodies, double *d_res, cudaStream_t st,
                    int *launches) const {
    if (n_bodies_ == 0)
        return SKB_OK;
    const BodyItem *items = (const BodyItem *)items_.ptr;
    const double *r = (const double *)r_.ptr, *c = (const double *)centers_.ptr, *w = (const double *)weights_.ptr,
                 *ex = (const double *)ex_.ptr, *ey = (const double *)ey_.ptr, *ez = (const double *)ez_.ptr;
    if (!windowed_) {
        body_matvec_kernel<false><<<(unsigned)n_bodies_, kBodyThreads, 0, st>>>(items, r, c, w, ex, ey, ez, d_x_bodies,
                                                                                d_v_bodies, d_res, 0, 0, 0);
        return launched(launches);
    }
    if (win_b1_ == win_b0_) // no body row is this member's
        return SKB_OK;
    body_matvec_kernel<true><<<(unsigned)(win_b1_ - win_b0_), kBodyThreads, 0, st>>>(
        items, r, c, w, ex, ey, ez, d_x_bodies, d_v_bodies, d_res, win_b0_, win_lo_, win_hi_);
    return launched(launches);
}

int skb::load_rhs_rows_kernel() {
    cudaFuncAttributes fa;
    CUDA_TRY(cudaFuncGetAttributes(&fa, system_rhs_rows_kernel));
    return SKB_OK;
}

int BodyOps::rhs_rows(bool bodies, const double *d_v_bodies, double *d_rhs_bodies, const double *d_v_shell,
                      long long n_shell_rows, double *d_rhs_shell, cudaStream_t st, int *launches) const {
    int b0 = 0, nb = 0;
    long long lo = 0, hi = 0;
    if (bodies && n_bodies_ > 0) {
        b0 = windowed_ ? win_b0_ : 0;
        nb = windowed_ ? win_b1_ - win_b0_ : n_bodies_;
        lo = windowed_ ? win_lo_ : 0;
        hi = windowed_ ? win_hi_ : LLONG_MAX;
    }
    const long long n3 = 3 * n_shell_rows;
    const int shell_ctas = (int)std::min<long long>((n3 + kBodyThreads - 1) / kBodyThreads, 1024);
    if (nb + shell_ctas == 0)
        return SKB_OK;
    system_rhs_rows_kernel<<<(unsigned)(nb + shell_ctas), kBodyThreads, 0, st>>>(
        (const BodyItem *)items_.ptr, b0, nb, lo, hi, d_v_bodies, d_rhs_bodies, d_v_shell, n3, d_rhs_shell);
    return launched(launches);
}

// BodyContainer::apply_preconditioner (body_container.cpp:510-521): A_LU_.solve(x) per body, here a GEMV over the
// explicit inverse (as for the fibers, skb_flow_set_fiber_preconditioner)
int BodyOps::precondition(const double *d_x, double *d_y, cudaStream_t st, int *launches) const {
    return launch_gemv((const FiberGemvItem *)gemv_items_.ptr, n_gemv_, (const double *)a_inv_.ptr, d_x, d_y,
                       gemv_smem_, st, launches);
}

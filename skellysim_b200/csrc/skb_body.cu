// skb_body.cu -- the bodies' per-timestep operators and the fiber-body links of a flow (BodyOps, skb_internal.hpp): their
// checks and uploads, and the launches of body_ops.cuh and of the body preconditioner's GEMV.  Knows nothing of skb_flow:
// skb_system.cu hands it the geometry, the fibers and their operators.
#include "body_ops.cuh"
#include "fiber_ops.cuh"
#include "skb_internal.hpp"

#include <algorithm>
#include <climits>
#include <cmath>
#include <vector>

using namespace skb;

struct BodyOps::Plan {
    std::vector<BodyItem> items;
    std::vector<FiberGemvItem> gemv;
    std::vector<PlaceBody> place; // the kept inverses, for body_place_kernel
    int n_bodies = 0, b0 = 0, b1 = 0, place_ctas = 0;
    long long nodes = 0, sol = 0;
    long long inv_first = 0, inv_own = 0; // the kept inverses, contiguous in the concatenated A_inv
    long long lo = 0, hi = -1;
    size_t smem = 0;
};

int BodyOps::plan(const char *who, const int *n_nodes, int n_bodies, long long n_body_nodes,
                  const double *node_weights, bool with_inverse, long long lo, long long hi, Plan &pl) const {
    const bool windowed = hi >= 0;
    pl.items.assign((size_t)n_bodies, BodyItem{});
    pl.n_bodies = n_bodies;
    pl.lo = lo, pl.hi = hi;
    long long nodes = 0, sol = 0, inv = 0;
    int max_cols = 0, b0 = n_bodies, b1 = 0;
    for (int b = 0; b < n_bodies; ++b) {
        const int n = n_nodes[b];
        if (n < 1)
            return set_error(SKB_ERR_INVALID, "%s: body %d has %d nodes", who, b, n);
        pl.items[(size_t)b] = BodyItem{nodes, sol, n, 0};
        const int m = 3 * n + 6;
        bool kept = !windowed;
        if (!windowed) {
            for (int r0 = 0; r0 < m; r0 += kFiberGemvRows)
                pl.gemv.push_back(FiberGemvItem{inv, sol, sol, m, m, r0, n, b, 0});
        } else if (nodes < hi && nodes + n > lo) {
            // the owned rows of this body: node rows [r_lo, r_hi), and [3n, 3n + 6) if its first node is owned; a
            // 32-row block that reaches any of them is evaluated (the other rows of the block are never read)
            if (b0 > b)
                b0 = b, pl.inv_first = inv;
            b1 = b + 1;
            const int r_lo = 3 * (int)(std::max(lo, nodes) - nodes), r_hi = 3 * (int)(std::min(hi, nodes + n) - nodes);
            const bool six = nodes >= lo;
            for (int r0 = 0; r0 < m; r0 += kFiberGemvRows) {
                const int r1 = r0 + kFiberGemvRows;
                if ((r0 < r_hi && r1 > r_lo) || (six && r1 > 3 * n))
                    pl.gemv.push_back(FiberGemvItem{inv - pl.inv_first, sol, sol, m, m, r0, n, b, 0});
            }
            pl.inv_own = inv + (long long)m * m - pl.inv_first;
            kept = true;
        }
        if (kept) {
            pl.place.push_back(PlaceBody{inv - pl.inv_first, m, b, pl.place_ctas, 0});
            pl.place_ctas += m / 3;
        }
        max_cols = std::max(max_cols, m);
        nodes += n;
        sol += m;
        inv += (long long)m * m;
    }
    if (!windowed)
        pl.inv_own = inv;
    if (nodes != n_body_nodes)
        return set_error(SKB_ERR_INVALID, "%s: the bodies' node counts sum to %lld, skb_flow_set_bodies has %lld nodes",
                         who, nodes, n_body_nodes);
    for (long long i = 0; i < nodes; ++i)
        if (!(node_weights[i] > 0))
            return set_error(SKB_ERR_INVALID, "%s: node_weights[%lld] = %g (must be > 0)", who, i, node_weights[i]);
    // fiber_gemv_kernel<0>: x (cols, rounded up to even) and the slice partials
    pl.smem = ((size_t)((max_cols + 1) & ~1) + kFiberGemvThreads) * sizeof(double);
    if (with_inverse && pl.smem > kFiberGemvSmemMax)
        return set_error(SKB_ERR_INVALID, "%s: a body of %d unknowns exceeds the shared memory of the preconditioner's "
                                          "GEMV", who, max_cols);
    pl.nodes = nodes;
    pl.sol = sol;
    pl.b0 = std::min(b0, b1);
    pl.b1 = b1;
    return SKB_OK;
}

// the geometry and the tables of a plan, and the per-matvec buffers; on st, not synchronised
int BodyOps::upload_layout(const Plan &pl, const double *r_body, const double *centers, const double *node_weights,
                           cudaStream_t st) {
    SKB_TRY(items_.upload(pl.items.data(), pl.items.size() * sizeof(BodyItem), st));
    SKB_TRY(r_.upload(r_body, (size_t)pl.nodes * 24, st));
    SKB_TRY(centers_.upload(centers, (size_t)pl.n_bodies * 24, st));
    SKB_TRY(weights_.upload(node_weights, (size_t)pl.nodes * 8, st));
    SKB_TRY(gemv_items_.upload(pl.gemv.data(), pl.gemv.size() * sizeof(FiberGemvItem), st));
    SKB_TRY(dens_.ensure((size_t)pl.nodes * 24 + 8));
    SKB_TRY(force_.ensure((size_t)pl.n_bodies * 24 + 8));
    return torque_.ensure((size_t)pl.n_bodies * 24 + 8);
}

void BodyOps::commit(const Plan &pl, bool with_inverse) {
    n_bodies_ = pl.n_bodies;
    sol_size_ = pl.sol;
    inv_own_ = with_inverse ? pl.inv_own : 0;
    windowed_ = pl.hi >= 0;
    win_b0_ = pl.b0;
    win_b1_ = pl.b1;
    win_lo_ = pl.lo;
    win_hi_ = pl.hi;
    n_gemv_ = (int)pl.gemv.size();
    gemv_smem_ = pl.smem;
    inv_set_ = with_inverse || pl.n_bodies == 0;
    ops_set_ = true;
}

// a group member's kernels are loaded when it is set up: a lazy load at the first launch would wait behind a peer on
// the same device spinning on a flag
static int load_member_kernels() {
    cudaFuncAttributes fa;
    CUDA_TRY(cudaFuncGetAttributes(&fa, fiber_link_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, body_sum_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, body_matvec_kernel<true>));
    return SKB_OK;
}

int BodyOps::set_operators(const int *n_nodes, int n_bodies, long long n_body_nodes, const double *r_body,
                           const double *centers, const double *node_weights, const double *ex, const double *ey,
                           const double *ez, const double *A_inv, cudaStream_t st, long long lo, long long hi) {
    Plan pl;
    SKB_TRY(plan("skb_flow_set_body_operators", n_nodes, n_bodies, n_body_nodes, node_weights, A_inv != nullptr, lo,
                 hi, pl));
    ops_set_ = inv_set_ = false;
    SKB_TRY(upload_layout(pl, r_body, centers, node_weights, st));
    SKB_TRY(ex_.upload(ex, (size_t)pl.nodes * 24, st));
    SKB_TRY(ey_.upload(ey, (size_t)pl.nodes * 24, st));
    SKB_TRY(ez_.upload(ez, (size_t)pl.nodes * 24, st));
    if (A_inv && pl.inv_own > 0) {
        SKB_TRY(a_inv_.ensure((size_t)pl.inv_own * 8));
        SKB_TRY(upload_pageable(a_inv_.ptr, A_inv + pl.inv_first, (size_t)pl.inv_own * 8, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st)); // the host tables above go out of scope
    if (hi >= 0)
        SKB_TRY(load_member_kernels());
    commit(pl, A_inv != nullptr);
    return SKB_OK;
}

int BodyOps::set_frames(const int *n_nodes, int n_bodies, long long n_body_nodes, const double *pos_ref,
                        const double *normal_ref, const double *node_weights, const double *ex0, const double *ey0,
                        const double *ez0, const double *A_inv0, cudaStream_t st, long long lo, long long hi) {
    Plan pl;
    SKB_TRY(plan("skb_flow_set_body_frames", n_nodes, n_bodies, n_body_nodes, node_weights, A_inv0 != nullptr, lo,
                 hi, pl));
    const size_t nodes = (size_t)pl.nodes;
    ops_set_ = inv_set_ = frames_set_ = false;
    // every buffer place writes, at its final size (place allocates nothing)
    SKB_TRY(ex0_.upload(ex0, nodes * 24, st));
    SKB_TRY(ey0_.upload(ey0, nodes * 24, st));
    SKB_TRY(ez0_.upload(ez0, nodes * 24, st));
    SKB_TRY(place_items_.upload(pl.place.data(), pl.place.size() * sizeof(PlaceBody), st));
    SKB_TRY(rot_.ensure((size_t)n_bodies * 72 + 8));
    SKB_TRY(items_.ensure(pl.items.size() * sizeof(BodyItem) + 8));
    SKB_TRY(r_.ensure(nodes * 24 + 8));
    SKB_TRY(centers_.ensure((size_t)n_bodies * 24 + 8));
    SKB_TRY(weights_.upload(node_weights, nodes * 8, st));
    SKB_TRY(gemv_items_.ensure(pl.gemv.size() * sizeof(FiberGemvItem) + 8));
    SKB_TRY(ex_.ensure(nodes * 24 + 8));
    SKB_TRY(ey_.ensure(nodes * 24 + 8));
    SKB_TRY(ez_.ensure(nodes * 24 + 8));
    SKB_TRY(dens_.ensure(nodes * 24 + 8));
    SKB_TRY(force_.ensure((size_t)n_bodies * 24 + 8));
    SKB_TRY(torque_.ensure((size_t)n_bodies * 24 + 8));
    if (A_inv0 && pl.inv_own > 0) {
        SKB_TRY(a_inv0_.ensure((size_t)pl.inv_own * 8));
        SKB_TRY(a_inv_.ensure((size_t)pl.inv_own * 8));
        SKB_TRY(upload_pageable(a_inv0_.ptr, A_inv0 + pl.inv_first, (size_t)pl.inv_own * 8, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    cudaFuncAttributes fa;
    CUDA_TRY(cudaFuncGetAttributes(&fa, body_place_kernel));
    if (hi >= 0)
        SKB_TRY(load_member_kernels());
    frame_n_.assign(n_nodes, n_nodes + n_bodies);
    frame_r_.assign(pos_ref, pos_ref + 3 * nodes);
    frame_nrm_.assign(normal_ref, normal_ref + 3 * nodes);
    frame_w_.assign(node_weights, node_weights + nodes);
    frame_lo_ = lo, frame_hi_ = hi;
    frame_inv_ = A_inv0 != nullptr;
    n_place_ = (int)pl.place.size();
    place_ctas_ = pl.place_ctas;
    frames_set_ = true;
    return SKB_OK;
}

void BodyOps::placed_geometry(const double *R, const double *centers, std::vector<double> &pos,
                              std::vector<double> &normals) const {
    pos.resize(frame_r_.size());
    normals.resize(frame_nrm_.size());
    long long g = 0;
    for (size_t b = 0; b < frame_n_.size(); ++b) {
        const double *Rb = R + 9 * b, *c = centers + 3 * b;
        for (int i = 0; i < frame_n_[b]; ++i, ++g) {
            const double *r = &frame_r_[3 * g], *n = &frame_nrm_[3 * g];
            for (int k = 0; k < 3; ++k) { // place(), body_spherical.cpp:146-159, with the rotation matrix
                pos[3 * g + k] = c[k] + (Rb[3 * k] * r[0] + Rb[3 * k + 1] * r[1] + Rb[3 * k + 2] * r[2]);
                normals[3 * g + k] = Rb[3 * k] * n[0] + Rb[3 * k + 1] * n[1] + Rb[3 * k + 2] * n[2];
            }
        }
    }
}

int BodyOps::place(const double *R, const double *r_body, const double *centers, cudaStream_t st) {
    Plan pl;
    SKB_TRY(plan("skb_flow_place_bodies", frame_n_.data(), (int)frame_n_.size(), frame_nodes(), frame_w_.data(),
                 frame_inv_, frame_lo_, frame_hi_, pl));
    ops_set_ = inv_set_ = false;
    // within the capacities set_frames gave (buffers only grow): nothing is allocated
    SKB_TRY(upload_layout(pl, r_body, centers, frame_w_.data(), st));
    SKB_TRY(rot_.upload(R, (size_t)pl.n_bodies * 72, st));
    const int n_inv_ctas = frame_inv_ ? place_ctas_ : 0;
    if (n_inv_ctas + pl.n_bodies > 0) {
        body_place_kernel<<<(unsigned)(n_inv_ctas + pl.n_bodies), kPlaceThreads, 0, st>>>(
            (const PlaceBody *)place_items_.ptr, n_place_, n_inv_ctas, (const BodyItem *)items_.ptr,
            (const double *)rot_.ptr, (const double *)a_inv0_.ptr, (double *)a_inv_.ptr, (const double *)ex0_.ptr,
            (const double *)ey0_.ptr, (const double *)ez0_.ptr, (double *)ex_.ptr, (double *)ey_.ptr,
            (double *)ez_.ptr);
        CUDA_TRY(cudaGetLastError());
        count_launch(1);
    }
    CUDA_TRY(cudaStreamSynchronize(st)); // the host tables above go out of scope
    commit(pl, frame_inv_);
    return SKB_OK;
}

int BodyOps::read(double *ex, double *ey, double *ez, double *A_inv, cudaStream_t st) const {
    const long long nodes = n_bodies_ > 0 ? sol_size_ / 3 - 2LL * n_bodies_ : 0; // sum(3 n + 6) = 3 N_b + 6 n_bodies
    double *dst[4] = {ex, ey, ez, A_inv};
    const DevBuf *src[4] = {&ex_, &ey_, &ez_, &a_inv_};
    for (int k = 0; k < 4; ++k) {
        const size_t bytes = k < 3 ? (size_t)nodes * 24 : (size_t)inv_own_ * 8;
        if (dst[k] && bytes > 0)
            CUDA_TRY(cudaMemcpyAsync(dst[k], src[k]->ptr, bytes, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
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
        SKB_TRY(link_fibers_.upload(lf.data(), lf.size() * sizeof(LinkFiber), st));
        SKB_TRY(csr_begin_.upload(count.data(), count.size() * sizeof(int), st));
        SKB_TRY(csr_fib_.upload(csr_fib.data(), csr_fib.size() * sizeof(int), st));
        SKB_TRY(link_.ensure((size_t)nfib * 56));
        SKB_TRY(contrib_.ensure((size_t)nfib * 48));
        CUDA_TRY(cudaStreamSynchronize(st)); // the host tables above go out of scope
    }
    n_fibers_ = nfib;
    any_bound_ = any;
    links_set_ = true;
    return SKB_OK;
}

int BodyOps::size_links(int n_fibers, int n_bodies) {
    const size_t nf = (size_t)std::max(n_fibers, 0);
    SKB_TRY(link_fibers_.ensure(nf * sizeof(LinkFiber)));
    SKB_TRY(csr_begin_.ensure(((size_t)std::max(n_bodies, 0) + 1) * sizeof(int)));
    SKB_TRY(csr_fib_.ensure(nf * sizeof(int)));
    SKB_TRY(link_.ensure(nf * 56));
    return contrib_.ensure(nf * 48);
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

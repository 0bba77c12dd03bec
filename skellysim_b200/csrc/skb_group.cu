// skb_group.cu -- one member of a multi-GPU group of flows (Group, skb_internal.hpp): its window, the window's set-up
// and exchange with the other members (CUDA IPC or peer access), and the steps of one matvec's protocol -- push, flag
// barriers, pull -- over the kernels of group_kernels.cuh.  Knows nothing of skb_flow: skb_flow.cu sets it up,
// skb_matvec.cu runs the steps.
#include "group_kernels.cuh"
#include "skb_internal.hpp"
#include "../../include/skelly_b200_flow.h"

#include <algorithm>
#include <cstring>

using namespace skb;

// a flag wait that outlasts this gives up and records the missing rank in the error word (~10 s at 2 GHz)
static constexpr unsigned long long kFlagTimeoutCycles = 20ULL * 1000 * 1000 * 1000;

int Group::init(int rank, int size, long long n_fib, long long n_pad_fib, long long n_shell, long long n_pad_shell,
                long long n_body, int n_bodies, int n_fibers) {
    *this = Group(); // the old window and mappings are released here
    if (size == 1)
        return SKB_OK;
    rank_ = rank;
    size_ = size;
    n_fib_ = n_fib;
    n_shell_ = n_shell;
    n_body_ = n_body;
    n_bodies_ = n_bodies;
    n_fibers_ = n_fibers;
    size_t off = 0;
    auto take = [&](size_t bytes) {
        const size_t at = off;
        off += (bytes + 255) & ~(size_t)255;
        return at;
    };
    lay_.flags = take((size_t)(kGroupPhases * kMaxGroup + 8) * 8);
    for (int b = 0; b < 2; ++b) {
        lay_.f_sl[b] = take((size_t)n_pad_fib * 24 + 16);
        lay_.f_shell[b] = take((size_t)n_pad_shell * 48 + 16);
        lay_.x_shell[b] = take((size_t)n_shell * 24 + 16);
        lay_.ft_part[b] = take((size_t)kMaxGroup * n_bodies * 48 + 16);
        lay_.x_body[b] = take((size_t)n_body * 24 + (size_t)n_bodies * 48 + 16);
        lay_.dots[b] = take((size_t)kMaxGroup * kDotsSlot * 8);
        lay_.r_step[b] = take((size_t)n_fib * 24 + (size_t)n_fibers * 16 + 16);
    }
    lay_.u_part = take((size_t)n_fib * 24 + 16);
    lay_.u_part_shell = take((size_t)n_shell * 24 + 16);
    lay_.bytes = off;
    CUDA_TRY(cudaMalloc(window_.out(), lay_.bytes));
    CUDA_TRY(cudaMemset(window_, 0, lay_.bytes)); // flags at epoch 0, strength pads zero for good
    // loaded now, not lazily at their first launch, which would wait behind a peer on this device spinning on a flag
    // (the warm-up's solo matvec does not run them)
    cudaFuncAttributes fa;
    CUDA_TRY(cudaFuncGetAttributes(&fa, group_flag_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, group_push_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, group_pull_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, group_ft_store_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, group_ft_reduce_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, group_rows_store_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, group_rows_compact_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, group_dots_store_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, group_dots_reduce_kernel));
    peer_[rank] = window_;
    return SKB_OK;
}

int Group::export_handle(void *handle) const {
    static_assert(sizeof(cudaIpcMemHandle_t) == SKB_FLOW_IPC_HANDLE_BYTES, "handle size");
    cudaIpcMemHandle_t h;
    CUDA_TRY(cudaIpcGetMemHandle(&h, window_));
    std::memcpy(handle, &h, sizeof(h));
    return SKB_OK;
}

int Group::import_handle(int peer_rank, const void *handle) {
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle, sizeof(h));
    CUDA_TRY(cudaIpcOpenMemHandle(ipc_[peer_rank].out(), h, cudaIpcMemLazyEnablePeerAccess));
    peer_[peer_rank] = ipc_[peer_rank];
    return SKB_OK;
}

int Group::connect(int peer_rank, const Group &peer, int dev, int peer_dev) {
    if (peer.lay_.bytes != lay_.bytes || peer.n_fib_ != n_fib_ || peer.n_shell_ != n_shell_ ||
        peer.n_body_ != n_body_ || peer.n_bodies_ != n_bodies_ || peer.n_fibers_ != n_fibers_)
        return set_error(SKB_ERR_INVALID, "skb_flow_group_connect: the two members were laid out for different geometries");
    if (peer_dev != dev) {
        int can = 0;
        CUDA_TRY(cudaDeviceCanAccessPeer(&can, dev, peer_dev));
        if (!can)
            return set_error(SKB_ERR_CUDA, "device %d cannot address device %d (no NVLink / P2P path)", dev, peer_dev);
        cudaError_t e = cudaDeviceEnablePeerAccess(peer_dev, 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled)
            (void)cudaGetLastError();
        else if (e != cudaSuccess)
            return set_error(SKB_ERR_CUDA, "cudaDeviceEnablePeerAccess(%d -> %d): %s", dev, peer_dev,
                             cudaGetErrorString(e));
    }
    peer_[peer_rank] = peer.window_;
    return SKB_OK;
}

int Group::missing_peer(int *missing) const {
    *missing = -1;
    if (!window_)
        return SKB_OK;
    unsigned long long w = 0;
    const unsigned long long *word = (const unsigned long long *)own(lay_.flags) + kGroupPhases * kMaxGroup;
    CUDA_TRY(cudaMemcpy(&w, word, 8, cudaMemcpyDeviceToHost));
    if (w)
        *missing = (int)(w - 1);
    return SKB_OK;
}

int Group::check_layout(long long n_fib, long long n_shell, long long n_body, int n_bodies, int n_fibers) const {
    if (n_fib_ != n_fib || n_shell_ != n_shell || n_body_ != n_body || n_bodies_ != n_bodies || n_fibers_ != n_fibers)
        return set_error(SKB_ERR_STATE, "group member: the geometry changed size since skb_flow_group_init "
                                        "(%lld/%lld fiber, %lld/%lld periphery, %lld/%lld body nodes, %d/%d bodies, "
                                        "%d/%d fibers); re-initialise the group", n_fib, n_fib_, n_shell, n_shell_,
                         n_body, n_body_, n_bodies, n_bodies_, n_fibers, n_fibers_);
    return SKB_OK;
}

int Group::windows(char **w) const {
    const int n = solo_ ? 1 : size_;
    for (int m = 0; m < n; ++m)
        w[m] = (char *)peer_[solo_ ? rank_ : m];
    return n;
}

int Group::connected() const {
    if (!solo_)
        for (int m = 0; m < size_; ++m)
            if (!peer_[m])
                return set_error(SKB_ERR_STATE, "group member %d: not all peers are connected (skb_flow_group_import / "
                                                "_connect)", rank_);
    return SKB_OK;
}

int Group::begin() {
    SKB_TRY(connected());
    epoch_ += 1; // the only place it advances
    return SKB_OK;
}

// pack + all-gather in one kernel
int Group::push(const double *d_fw, const double *d_weight, long long fa, long long n_f, const double *d_density,
                const double *d_normal, long long sa, long long n_s, double two_eta, int num_sms, cudaStream_t st,
                int *launches) const {
    const int par = (int)(epoch_ & 1);
    GroupPushArgs a;
    a.fw = d_fw;
    a.weight = d_weight;
    a.fa = fa;
    a.n_f = n_f;
    a.density = d_density;
    a.normal = d_normal;
    a.sa = sa;
    a.n_s = n_s;
    a.two_eta = two_eta;
    char *w[kMaxGroup];
    a.size = windows(w);
    for (int m = 0; m < a.size; ++m) {
        a.f_sl[m] = (double *)(w[m] + lay_.f_sl[par]);
        a.f_shell[m] = (double *)(w[m] + lay_.f_shell[par]);
        a.x_shell[m] = (double *)(w[m] + lay_.x_shell[par]);
    }
    const long long work = 3 * n_f + n_s;
    if (work == 0)
        return SKB_OK;
    const unsigned nblk = (unsigned)std::min<long long>((work + 255) / 256, 4LL * num_sms);
    group_push_kernel<<<nblk, 256, 0, st>>>(a);
    return launched(launches);
}

// signal: this member's stores so far have landed in every window; wait: every member's have landed in this one
int Group::barrier(int phase, bool signal, bool wait, cudaStream_t st, int *launches) const {
    if (solo_)
        return SKB_OK;
    GroupFlagArgs a;
    for (int m = 0; m < size_; ++m)
        a.flags[m] = (unsigned long long *)((char *)peer_[m] + lay_.flags);
    a.rank = rank_;
    a.size = size_;
    a.phase = phase;
    a.epoch = epoch_;
    a.do_signal = signal;
    a.do_wait = wait;
    a.timeout_cycles = kFlagTimeoutCycles;
    group_flag_kernel<<<1, 32, 0, st>>>(a);
    return launched(launches);
}

// this member's partial forces / torques into its slot of every window (before barrier 0)
int Group::push_forces(const double *d_f, const double *d_t, cudaStream_t st, int *launches) const {
    if (n_bodies_ == 0)
        return SKB_OK;
    const size_t off = lay_.ft_part[epoch_ & 1] + (size_t)rank_ * n_bodies_ * 48;
    GroupFtStoreArgs a;
    a.f = d_f;
    a.t = d_t;
    a.n3 = 3 * n_bodies_;
    char *w[kMaxGroup];
    a.size = windows(w);
    for (int m = 0; m < a.size; ++m)
        a.slot[m] = (double *)(w[m] + off);
    group_ft_store_kernel<<<(unsigned)((2 * a.n3 + 255) / 256), 256, 0, st>>>(a);
    return launched(launches);
}

// the totals out of this member's window, slots in rank order (after barrier 0); solo: the own partial only
int Group::reduce_forces(double *d_f, double *d_t, cudaStream_t st, int *launches) const {
    if (n_bodies_ == 0)
        return SKB_OK;
    GroupFtReduceArgs a;
    a.slots = own(lay_.ft_part[epoch_ & 1]);
    a.stride = 6LL * n_bodies_;
    a.first = solo_ ? rank_ : 0;
    a.count = solo_ ? 1 : size_;
    a.n3 = 3 * n_bodies_;
    a.f = d_f;
    a.t = d_t;
    group_ft_reduce_kernel<<<(unsigned)((2 * a.n3 + 255) / 256), 256, 0, st>>>(a);
    return launched(launches);
}

// one epoch of its own: begin, the store into this member's slot of every window, the dots phase, the rank-order sum
int Group::reduce_dots(double *d_v, int m, cudaStream_t st, int *launches) {
    if (m > kDotsSlot)
        return set_error(SKB_ERR_INVALID, "group member %d: %d dots exceed the window's slot of %d", rank_, m, kDotsSlot);
    SKB_TRY(begin());
    const int par = (int)(epoch_ & 1);
    GroupDotsStoreArgs a;
    a.v = d_v;
    a.m = m;
    char *w[kMaxGroup];
    a.size = windows(w);
    for (int k = 0; k < a.size; ++k)
        a.slot[k] = (double *)(w[k] + lay_.dots[par]) + (size_t)rank_ * kDotsSlot;
    const unsigned blocks = (unsigned)((m + 255) / 256);
    group_dots_store_kernel<<<blocks, 256, 0, st>>>(a);
    SKB_TRY(launched(launches));
    SKB_TRY(barrier(kDotsPhase, true, true, st, launches));
    group_dots_reduce_kernel<<<blocks, 256, 0, st>>>(own(lay_.dots[par]), kDotsSlot, solo_ ? rank_ : 0,
                                                     solo_ ? 1 : size_, m, d_v);
    return launched(launches);
}

// reduce-scatter fused with the accumulation
int Group::pull(Partials which, long long row0, long long n_rows, double *d_v, cudaStream_t st, int *launches) const {
    if (n_rows == 0)
        return SKB_OK;
    const size_t off = which == kFiberRows ? lay_.u_part : lay_.u_part_shell;
    GroupPullArgs a;
    char *w[kMaxGroup];
    a.size = windows(w);
    for (int m = 0; m < a.size; ++m)
        a.u_part[m] = (const double *)(w[m] + off);
    a.fa = row0;
    a.n_f = n_rows;
    a.v = d_v;
    a.accumulate = 1;
    group_pull_kernel<<<(unsigned)((3 * n_rows + 255) / 256), 256, 0, st>>>(a);
    return launched(launches);
}

int Group::step_windows(double **r_step) const {
    char *w[kMaxGroup];
    const int n = windows(w);
    for (int m = 0; m < n; ++m)
        r_step[m] = (double *)(w[m] + lay_.r_step[epoch_ & 1]);
    return n;
}

// ---- a rank-per-GPU member's own rows of the solution vector ----

bool skb::body_row_pieces(const int *n_nodes, int n_bodies, long long b0, long long b1, std::vector<RowPiece> &out) {
    out.clear();
    long long local = 0;
    auto add = [&](long long a, long long e) { // body-part entries [a, e)
        if (e <= a)
            return;
        if (!out.empty() && out.back().body + out.back().len == a)
            out.back().len += e - a;
        else
            out.push_back(RowPiece{local, a, e - a});
        local += e - a;
    };
    long long node = 0, sol = 0;
    for (int b = 0; b < n_bodies; ++b) {
        const long long n = n_nodes[b];
        add(sol + 3 * (std::max(b0, node) - node), sol + 3 * (std::min(b1, node + n) - node));
        if (node >= b0 && node < b1)
            add(sol + 3 * n, sol + 3 * n + 6);
        node += n;
        sol += 3 * n + 6;
    }
    return out.size() <= (size_t)kMaxRowPieces;
}

void Group::set_body_rows(const std::vector<RowPiece> &pieces, const Ranges &ranges) {
    rows_ = Rows();
    for (const RowPiece &p : pieces) {
        rows_.local[rows_.n] = p.local;
        rows_.body[rows_.n] = p.body;
        rows_.len[rows_.n] = p.len;
        rows_.n += 1;
        rows_.total += p.len;
    }
    rows_set_ = true;
    rows_ranges_ = ranges;
}

static RowPiecesDev pieces_dev(const long long *local, const long long *body, const long long *len, int n,
                               long long total) {
    RowPiecesDev p;
    for (int k = 0; k < kMaxRowPieces; ++k) {
        p.local[k] = k < n ? local[k] : 0;
        p.body[k] = k < n ? body[k] : 0;
        p.len[k] = k < n ? len[k] : 0;
    }
    p.n = n;
    p.total = total;
    return p;
}

// the own rows into every window (before the rows phase's barrier)
int Group::store_rows(const double *d_body, const double *d_shell, long long sa, long long n_s, int num_sms,
                      cudaStream_t st, int *launches) const {
    const int par = (int)(epoch_ & 1);
    GroupRowsStoreArgs a;
    a.pieces = pieces_dev(rows_.local, rows_.body, rows_.len, rows_.n, rows_.total);
    a.body = d_body;
    a.shell = d_shell;
    a.shell_off = 3 * sa;
    a.n_shell3 = d_shell ? 3 * n_s : 0;
    char *w[kMaxGroup];
    a.size = windows(w);
    for (int m = 0; m < a.size; ++m) {
        a.x_body[m] = (double *)(w[m] + lay_.x_body[par]);
        a.x_shell[m] = (double *)(w[m] + lay_.x_shell[par]);
    }
    const long long work = a.pieces.total + a.n_shell3;
    if (work == 0)
        return SKB_OK;
    const unsigned nblk = (unsigned)std::min<long long>((work + 255) / 256, 4LL * num_sms);
    group_rows_store_kernel<<<nblk, 256, 0, st>>>(a);
    return launched(launches);
}

int Group::rows_barrier(bool signal, bool wait, cudaStream_t st, int *launches) const {
    return barrier(kRowsPhase, signal, wait, st, launches);
}

int Group::compact_rows(const double *d_full, double *d_local, cudaStream_t st, int *launches) const {
    if (rows_.total == 0)
        return SKB_OK;
    GroupRowsCompactArgs a;
    a.pieces = pieces_dev(rows_.local, rows_.body, rows_.len, rows_.n, rows_.total);
    a.full = d_full;
    a.local = d_local;
    group_rows_compact_kernel<<<(unsigned)((rows_.total + 255) / 256), 256, 0, st>>>(a);
    return launched(launches);
}

// host-only: the pieces a rank-per-GPU member's local vector is laid out by
extern "C" int skb_group_body_pieces(const int *n_nodes, int n_bodies, int64_t body_begin, int64_t body_end,
                                     int64_t *pieces, int max_pieces, int *n_pieces) {
    if (n_bodies < 0 || (n_bodies > 0 && !n_nodes) || body_begin < 0 || body_end < body_begin || !n_pieces ||
        max_pieces < 0 || (max_pieces > 0 && !pieces))
        return set_error(SKB_ERR_INVALID, "skb_group_body_pieces: bad arguments");
    for (int b = 0; b < n_bodies; ++b)
        if (n_nodes[b] < 1)
            return set_error(SKB_ERR_INVALID, "skb_group_body_pieces: body %d has %d nodes", b, n_nodes[b]);
    std::vector<RowPiece> out;
    body_row_pieces(n_nodes, n_bodies, body_begin, body_end, out);
    *n_pieces = (int)out.size();
    if ((int)out.size() > max_pieces)
        return set_error(SKB_ERR_INVALID, "skb_group_body_pieces: %d pieces, room for %d", (int)out.size(), max_pieces);
    for (size_t k = 0; k < out.size(); ++k) {
        pieces[3 * k + 0] = out[k].local;
        pieces[3 * k + 1] = out[k].body;
        pieces[3 * k + 2] = out[k].len;
    }
    return SKB_OK;
}

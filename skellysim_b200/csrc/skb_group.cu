// skb_group.cu -- one member of a multi-GPU group of flows (Group, skb_internal.hpp): its window, the window's set-up
// and exchange with the other members (CUDA IPC or peer access), and the steps of one matvec's protocol -- push, flag
// barriers, pull -- over the kernels of group_kernels.cuh.  Knows nothing of skb_flow: skb_matvec.cu runs the steps.
#include "group_kernels.cuh"
#include "skb_internal.hpp"
#include "../../include/skelly_b200_flow.h"

#include <algorithm>
#include <cstring>

using namespace skb;

// a flag wait that outlasts this gives up and records the missing rank in the error word (~10 s at 2 GHz)
static constexpr unsigned long long kFlagTimeoutCycles = 20ULL * 1000 * 1000 * 1000;

static int launched(int *launches) {
    CUDA_TRY(cudaGetLastError());
    count_launch(1);
    *launches += 1;
    return SKB_OK;
}

int Group::init(int rank, int size, long long n_fib, long long n_pad_fib, long long n_shell, long long n_pad_shell,
                int n_bodies) {
    *this = Group(); // the old window and mappings are released here
    if (size == 1)
        return SKB_OK;
    rank_ = rank;
    size_ = size;
    n_fib_ = n_fib;
    n_shell_ = n_shell;
    n_bodies_ = n_bodies;
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
    }
    lay_.u_part = take((size_t)n_fib * 24 + 16);
    lay_.u_part_shell = take((size_t)n_shell * 24 + 16);
    lay_.bytes = off;
    CUDA_TRY(cudaMalloc(window_.out(), lay_.bytes));
    CUDA_TRY(cudaMemset(window_, 0, lay_.bytes)); // flags at epoch 0, strength pads zero for good
    // loaded now, not lazily at their first launch, which would wait behind a peer on this device spinning on a flag
    // (the warm-up's solo matvec does not run them)
    cudaFuncAttributes fa;
    CUDA_TRY(cudaFuncGetAttributes(&fa, group_ft_store_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, group_ft_reduce_kernel));
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
        peer.n_bodies_ != n_bodies_)
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

int Group::check_layout(long long n_fib, long long n_shell, int n_bodies) const {
    if (n_fib_ != n_fib || n_shell_ != n_shell || n_bodies_ != n_bodies)
        return set_error(SKB_ERR_STATE, "group member: the geometry changed size since skb_flow_group_init "
                                        "(%lld/%lld fiber, %lld/%lld periphery nodes, %d/%d bodies); re-initialise the "
                                        "group", n_fib, n_fib_, n_shell, n_shell_, n_bodies, n_bodies_);
    return SKB_OK;
}

int Group::windows(char **w) const {
    const int n = solo_ ? 1 : size_;
    for (int m = 0; m < n; ++m)
        w[m] = (char *)peer_[solo_ ? rank_ : m];
    return n;
}

int Group::begin() {
    if (!solo_)
        for (int m = 0; m < size_; ++m)
            if (!peer_[m])
                return set_error(SKB_ERR_STATE, "group member %d: not all peers are connected (skb_flow_group_import / "
                                                "_connect)", rank_);
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

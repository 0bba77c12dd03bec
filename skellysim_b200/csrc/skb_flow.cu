// skb_flow.cu -- the flow object (include/skelly_b200_flow.h): its lifetime, the geometry setters (fibers, periphery,
// bodies, point sources, background flow), the knobs of the matvec (cross kernel, overlap, self exclusion, target
// window and ranges), the statistics and host transfers every call frames its work with, the own fibers, and group
// membership.  The evaluations and the matvec that run on it are skb_matvec.cu.
#include "skb_flow.hpp"

#include <algorithm>
#include <cstdlib>
#include <memory>
#include <vector>

using namespace skb;

int skb::upload(skb_flow *fl, DevBuf &buf, const double *h, size_t n_doubles) {
    return buf.upload(h, n_doubles * 8, fl->stream);
}
int skb::download(skb_flow *fl, double *h, const DevBuf &buf, size_t n_doubles) {
    if (n_doubles > 0)
        CUDA_TRY(cudaMemcpyAsync(h, buf.ptr, n_doubles * 8, cudaMemcpyDeviceToHost, fl->stream));
    return SKB_OK;
}

int skb::stage_slots(std::vector<DevBuf> &slots, Transfers &x) {
    slots.resize(std::max(slots.size(), x.up.size() + x.down.size()));
    size_t k = 0;
    for (std::vector<Transfer> *list : {&x.up, &x.down})
        for (Transfer &t : *list) {
            DevBuf &slot = slots[k++];
            if (t.dev)
                continue;
            long long n = 0;
            for (const Run &r : t.runs)
                n = std::max(n, r.at + r.len);
            SKB_TRY(slot.ensure((size_t)n * 8 + 8));
            t.dev = (double *)slot.ptr;
        }
    return SKB_OK;
}

int skb::issue(const std::vector<Transfer> &list, bool upload, cudaStream_t st) {
    for (const Transfer &t : list)
        for (const Run &r : t.runs) {
            if (!t.host || !r.len)
                continue;
            double *d = t.dev + r.at, *h = t.host + r.whole;
            const size_t bytes = (size_t)r.len * 8;
            CUDA_TRY(upload ? cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st)
                            : cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, st));
        }
    return SKB_OK;
}

void skb::begin_stats(skb_flow *fl) {
    fl->launches = 0;
    fl->pairs = 0;
}
int skb::finish_stats(skb_flow *fl) {
    CUDA_TRY(cudaStreamSynchronize(fl->stream));
    float a = 0, b = 0;
    cudaEventElapsedTime(&a, fl->ev0, fl->ev1);
    cudaEventElapsedTime(&b, fl->evt0, fl->evt1);
    fl->stats.device_ms = a;
    fl->stats.total_ms = b;
    fl->stats.n_pairs = fl->pairs;
    fl->stats.launches = fl->launches;
    return SKB_OK;
}

int skb::device_stats(skb_flow *fl) {
    fl->stats.device_ms = fl->stats.total_ms = 0;
    fl->stats.n_pairs = fl->pairs;
    fl->stats.launches = fl->launches;
    return SKB_OK;
}

int skb::own_fibers(skb_flow *fl, const char *who, OwnFibers &own) {
    SKB_TRY(prepare_matvec_targets(fl));
    int f0 = 0, f1 = 0;
    if (fl->n_fibers > 0) {
        const auto &off = fl->h_fiber_off;
        f0 = (int)(std::lower_bound(off.begin(), off.end(), fl->fa) - off.begin());
        f1 = (int)(std::lower_bound(off.begin(), off.end(), fl->fb) - off.begin());
        if (off[(size_t)f0] != fl->fa || off[(size_t)f1] != fl->fb)
            return set_error(SKB_ERR_INVALID, "%s: the target window [%lld, %lld) cuts a fiber; use "
                                              "skb_flow_set_target_ranges (whole fibers)", who, fl->fa, fl->fb);
    }
    own = OwnFibers{f0, f1, fl->h_fiber_n.data(), fl->h_fiber_off.data(), (const double *)fl->r_fib.ptr,
                    (const double *)fl->fiber_length.ptr, fl->stream};
    return SKB_OK;
}

extern "C" {

int skb_flow_create(int device, skb_flow **out) {
    if (!out)
        return set_error(SKB_ERR_INVALID, "skb_flow_create: out == NULL");
    *out = nullptr;
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0)
        return set_error(SKB_ERR_NO_DEVICE, "no CUDA device available; this library has no CPU fallback");
    if (device < 0 || device >= n_dev)
        return set_error(SKB_ERR_INVALID, "skb_flow_create: device %d out of range (%d visible)", device, n_dev);
    std::unique_ptr<skb_flow> fl(new skb_flow);
    fl->dev = device;
    CUDA_TRY(cudaSetDevice(device));
    CUDA_TRY(cudaStreamCreateWithFlags(fl->stream.out(), cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreate(fl->ev0.out()));
    CUDA_TRY(cudaEventCreate(fl->ev1.out()));
    CUDA_TRY(cudaEventCreate(fl->evt0.out()));
    CUDA_TRY(cudaEventCreate(fl->evt1.out()));
    if (const char *e = getenv("SKB_GRAPHS"))
        fl->graphs_enabled = atoi(e) != 0;
    if (const char *e = getenv("SKB_OVERLAP")) // A/B switch of skb_flow_set_overlap's default
        fl->bg.enabled = atoi(e) != 0;
    SKB_TRY(prepare_device(device));
    const DeviceInfo di = query_device(device);
    // empty classes until set_* is called
    for (int k = 0; k < 2; ++k) {
        for (Evaluator *e : {&fl->fib[k], &fl->shell[k], &fl->body[k]})
            SKB_TRY(e->init(di));
        SKB_TRY(fl->fib[k].set_sources(SKB_STOKESLET, nullptr, 0, false, fl->stream));
        SKB_TRY(fl->shell[k].set_sources(SKB_STRESSLET, nullptr, 0, false, fl->stream));
        SKB_TRY(fl->body[k].set_sources(SKB_STRESSLET, nullptr, 0, false, fl->stream));
        SKB_TRY(fl->body[k].set_sources(SKB_STOKESLET, nullptr, 0, false, fl->stream));
    }
    *out = fl.release();
    return SKB_OK;
}

int skb_flow_destroy(skb_flow *fl) {
    if (!fl)
        return SKB_OK;
    cudaSetDevice(fl->dev);
    cudaStreamSynchronize(fl->stream);
    delete fl;
    return SKB_OK;
}

int skb_flow_set_fibers(skb_flow *fl, const double *r_fib, const int *n_nodes, const double *length, int n_fibers) {
    if (!fl || n_fibers < 0 || (n_fibers > 0 && (!r_fib || !n_nodes || !length)))
        return set_error(SKB_ERR_INVALID, "skb_flow_set_fibers: bad arguments");
    std::vector<long long> off((size_t)n_fibers + 1, 0);
    int max_n = 0;
    for (int f = 0; f < n_fibers; ++f) {
        if (n_nodes[f] < 2)
            return set_error(SKB_ERR_INVALID, "fiber %d has %d nodes (need >= 2)", f, n_nodes[f]);
        off[f + 1] = off[f] + n_nodes[f];
        max_n = std::max(max_n, n_nodes[f]);
    }
    if ((size_t)max_n * 48 > 200 * 1024)
        return set_error(SKB_ERR_INVALID, "fiber with %d nodes exceeds the shared-memory self-term kernel", max_n);
    fl->n_fibers = n_fibers;
    fl->n_fib = off[n_fibers];
    fl->max_fiber_nodes = max_n;
    fl->h_r_fib.assign(r_fib, r_fib + 3 * fl->n_fib);
    fl->h_fiber_n.assign(n_nodes, n_nodes + n_fibers);
    fl->h_fiber_len.assign(length, length + n_fibers);
    fl->h_fiber_off = off;
    fl->ops.invalidate(); // operators belong to one set of fibers
    fl->bodies.drop_links(); // ... and so do the links
    fl->mv_dirty = true;
    fl->geom_version++;
    CUDA_TRY(cudaSetDevice(fl->dev));
    for (int k = 0; k < 2; ++k)
        SKB_TRY(fl->fib[k].set_sources(SKB_STOKESLET, r_fib, fl->n_fib, false, fl->stream));
    if (n_fibers == 0)
        return SKB_OK;
    SKB_TRY(fl->fiber_offset.upload(off.data(), off.size() * 8, fl->stream));
    SKB_TRY(fl->fiber_length.upload(length, (size_t)n_fibers * 8, fl->stream));
    SKB_TRY(fl->r_fib.upload(r_fib, (size_t)fl->n_fib * 24, fl->stream));
    SKB_TRY(install_fiber_sources(fl));
    CUDA_TRY(cudaStreamSynchronize(fl->stream));
    return SKB_OK;
}

int skb_flow_set_periphery(skb_flow *fl, const double *node_pos, const double *node_normal, int64_t n_nodes) {
    if (!fl || n_nodes < 0 || (n_nodes > 0 && (!node_pos || !node_normal)))
        return set_error(SKB_ERR_INVALID, "skb_flow_set_periphery: bad arguments");
    fl->n_shell = n_nodes;
    fl->h_r_shell.assign(node_pos, node_pos + 3 * n_nodes);
    fl->mv_dirty = true;
    fl->geom_version++;
    CUDA_TRY(cudaSetDevice(fl->dev));
    for (int k = 0; k < 2; ++k) {
        SKB_TRY(fl->shell[k].set_sources(SKB_STRESSLET, node_pos, n_nodes, false, fl->stream));
        SKB_TRY(fl->shell[k].set_normals(node_normal, n_nodes, fl->stream));
    }
    CUDA_TRY(cudaStreamSynchronize(fl->stream));
    return SKB_OK;
}

int skb_flow_set_bodies(skb_flow *fl, const double *node_pos, const double *node_normal, int64_t n_nodes,
                        const double *centers, int n_bodies) {
    if (!fl || n_nodes < 0 || n_bodies < 0 || (n_nodes > 0 && (!node_pos || !node_normal)) ||
        (n_bodies > 0 && !centers) || (n_bodies == 0 && n_nodes > 0))
        return set_error(SKB_ERR_INVALID, "skb_flow_set_bodies: bad arguments");
    fl->n_body = n_nodes;
    fl->n_bodies = n_bodies;
    fl->h_r_body.assign(node_pos, node_pos + 3 * n_nodes);
    fl->h_centers.assign(centers, centers + 3 * (size_t)n_bodies);
    fl->placed = false; // skb_flow_place_bodies sets it again after this call
    fl->bodies.drop_operators(); // the bodies' operators and the nucleation sites belong to one placement
    fl->bodies.drop_links();
    fl->mv_dirty = true;
    fl->geom_version++;
    CUDA_TRY(cudaSetDevice(fl->dev));
    for (int k = 0; k < 2; ++k) {
        SKB_TRY(fl->body[k].set_sources(SKB_STRESSLET, node_pos, n_nodes, false, fl->stream));
        SKB_TRY(fl->body[k].set_normals(node_normal, n_nodes, fl->stream));
        SKB_TRY(fl->body[k].set_sources(SKB_STOKESLET, centers, n_bodies, false, fl->stream));
    }
    if (n_bodies > 0)
        SKB_TRY(fl->centers.upload(centers, (size_t)n_bodies * 24, fl->stream));
    CUDA_TRY(cudaStreamSynchronize(fl->stream));
    return SKB_OK;
}

int skb_flow_set_point_sources(skb_flow *fl, const double *positions, const double *forces, const double *torques,
                               int n_points) {
    if (!fl || n_points < 0 || (n_points > 0 && (!positions || !forces || !torques)))
        return set_error(SKB_ERR_INVALID, "skb_flow_set_point_sources: bad arguments");
    fl->n_points = n_points;
    fl->geom_version++;
    if (n_points == 0)
        return SKB_OK;
    CUDA_TRY(cudaSetDevice(fl->dev));
    SKB_TRY(fl->pt_pos.upload(positions, (size_t)n_points * 24, fl->stream));
    SKB_TRY(fl->pt_force.upload(forces, (size_t)n_points * 24, fl->stream));
    SKB_TRY(fl->pt_torque.upload(torques, (size_t)n_points * 24, fl->stream));
    CUDA_TRY(cudaStreamSynchronize(fl->stream));
    return SKB_OK;
}

int skb_flow_set_background(skb_flow *fl, const int *components, const double *scale_factor, const double *uniform) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_background: NULL");
    fl->geom_version++;
    if (!components || !scale_factor || !uniform) {
        fl->has_background = false;
        return SKB_OK;
    }
    for (int j = 0; j < 3; ++j) {
        if (components[j] < 0 || components[j] > 2)
            return set_error(SKB_ERR_INVALID, "skb_flow_set_background: components must be 0, 1 or 2");
        fl->bg_comp[j] = components[j];
        fl->bg_scale[j] = scale_factor[j];
        fl->bg_uniform[j] = uniform[j];
    }
    fl->has_background = true;
    return SKB_OK;
}

// ---- group membership (multi-GPU through peer memory, skb_group.cu) ----------------------------------------------
int skb_flow_group_init(skb_flow *fl, int rank, int size) {
    if (!fl || size < 1 || size > kMaxGroup || rank < 0 || rank >= size)
        return set_error(SKB_ERR_INVALID, "skb_flow_group_init: need 0 <= rank < size <= %d", kMaxGroup);
    CUDA_TRY(cudaSetDevice(fl->dev));
    CUDA_TRY(cudaStreamSynchronize(fl->stream));
    fl->mv_dirty = true;
    fl->ops.invalidate();
    fl->geom_version++;
    // the same padded sizes the evaluators use (Evaluator::set_sources): the window replaces their f_packed
    const long long n_pad_fib = fl->n_fib > 0 ? fl->fib[1].src[SKB_STOKESLET].n_pad : 0;
    const long long n_pad_shell = fl->n_shell > 0 ? fl->shell[1].src[SKB_STRESSLET].n_pad : 0;
    return fl->grp.init(rank, size, fl->n_fib, n_pad_fib, fl->n_shell, n_pad_shell, fl->n_body, fl->n_bodies,
                        fl->n_fibers);
}

int skb_flow_group_export(skb_flow *fl, void *handle) {
    if (!fl || !handle || !fl->grp.has_window())
        return set_error(SKB_ERR_INVALID, "skb_flow_group_export: no group window (skb_flow_group_init with size > 1 first)");
    CUDA_TRY(cudaSetDevice(fl->dev));
    return fl->grp.export_handle(handle);
}

int skb_flow_group_import(skb_flow *fl, int peer_rank, const void *handle) {
    if (!fl || !handle || !fl->grp.has_window() || peer_rank < 0 || peer_rank >= fl->grp.size() ||
        peer_rank == fl->grp.rank())
        return set_error(SKB_ERR_INVALID, "skb_flow_group_import: bad arguments");
    CUDA_TRY(cudaSetDevice(fl->dev));
    return fl->grp.import_handle(peer_rank, handle);
}

int skb_flow_group_connect(skb_flow *fl, int peer_rank, skb_flow *peer) {
    if (!fl || !peer || !fl->grp.has_window() || !peer->grp.has_window() || peer_rank < 0 ||
        peer_rank >= fl->grp.size() || peer_rank == fl->grp.rank() || peer->grp.rank() != peer_rank ||
        peer->grp.size() != fl->grp.size())
        return set_error(SKB_ERR_INVALID, "skb_flow_group_connect: bad arguments");
    CUDA_TRY(cudaSetDevice(fl->dev));
    return fl->grp.connect(peer_rank, peer->grp, fl->dev, peer->dev);
}

// One matvec of this member alone (no flags, own window only, zero strengths): every buffer of the path reaches its
// steady-state size, so that no cudaMalloc / cudaFree -- which synchronise the whole DEVICE -- happens later while a
// peer on the same device sits in a flag wait.  Needed when members share a GPU; harmless otherwise.
int skb_flow_group_warmup(skb_flow *fl) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_group_warmup: NULL flow");
    if (!fl->grp.member())
        return SKB_OK;
    CUDA_TRY(cudaSetDevice(fl->dev));
    SKB_TRY(prepare_matvec_targets(fl));
    const long long n_fw = fl->fb - fl->fa, n_sw = fl->sb - fl->sa;
    DevBuf z;
    const size_t n_z = (size_t)std::max<long long>({4 * n_fw, 3 * n_sw, 3 * fl->n_body, 3LL * fl->n_bodies, 1LL});
    SKB_TRY(z.ensure(n_z * 8));
    CUDA_TRY(cudaMemsetAsync(z.ptr, 0, n_z * 8, fl->stream));
    SKB_TRY(fl->vel.ensure((size_t)fl->n_win * 24 + 8));
    SKB_TRY(fl->fw.ensure((size_t)n_fw * 24 + 8));
    if (n_sw > 0 && fl->bg.enabled)
        SKB_TRY(overlap_buffers(fl, 3 * n_sw));
    fl->cur = fl->stream;
    fl->grp.set_solo(true);
    const double *zp = (const double *)z.ptr;
    int rc = matvec_core(fl, zp, zp, zp, zp, zp, 1.0, (double *)fl->vel.ptr);
    fl->grp.set_solo(false);
    cudaError_t e = cudaStreamSynchronize(fl->stream);
    fl->grp.restart();
    if (rc != SKB_OK)
        return rc;
    if (e != cudaSuccess)
        return set_error(SKB_ERR_CUDA, "skb_flow_group_warmup: %s", cudaGetErrorString(e));
    return SKB_OK;
}

// Profiling aid: evaluate this member's share ALONE from now on (no flags, own window only) -- the per-rank device time
// of an n-way group on one GPU.  Results are the member's partial view, not the group's.
int skb_flow_group_set_solo(skb_flow *fl, int solo) {
    if (!fl || !fl->grp.member())
        return set_error(SKB_ERR_INVALID, "skb_flow_group_set_solo: not a group member");
    fl->grp.set_solo(solo != 0);
    return SKB_OK;
}

int skb_flow_group_error(skb_flow *fl, int *missing_peer) {
    if (!fl || !missing_peer)
        return set_error(SKB_ERR_INVALID, "skb_flow_group_error: NULL");
    CUDA_TRY(cudaSetDevice(fl->dev));
    return fl->grp.missing_peer(missing_peer);
}

// ---- the knobs of the matvec -------------------------------------------------------------------------------------
int skb_flow_set_cross(skb_flow *fl, int mode) {
    if (!fl || mode < -1 || mode > 1)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_cross: mode must be -1 (auto), 0 (off) or 1 (on)");
    fl->cross_mode = mode;
    fl->mv_dirty = true;
    fl->geom_version++;
    return SKB_OK;
}

int skb_flow_set_overlap(skb_flow *fl, int on) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_overlap: NULL flow");
    fl->bg.enabled = on != 0;
    return SKB_OK;
}

int skb_flow_set_self_exclusion(skb_flow *fl, int fused) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_self_exclusion: NULL flow");
    fl->self_excl = fused != 0;
    fl->mv_dirty = true;
    fl->geom_version++;
    return SKB_OK;
}

int skb_flow_set_target_window(skb_flow *fl, int64_t begin, int64_t end) {
    if (!fl || begin < 0 || (end >= 0 && end < begin))
        return set_error(SKB_ERR_INVALID, "skb_flow_set_target_window: bad window [%lld, %lld)", (long long)begin,
                         (long long)end);
    fl->win_begin = begin;
    fl->win_end = end;
    fl->use_ranges = false;
    fl->mv_dirty = true;
    fl->ops.invalidate(); // resident fiber operators belong to one set of fiber rows
    fl->geom_version++;
    return SKB_OK;
}

int skb_flow_set_target_ranges(skb_flow *fl, int fiber_begin, int fiber_end, int64_t shell_begin, int64_t shell_end,
                               int64_t body_begin, int64_t body_end) {
    if (!fl || fiber_begin < 0 || fiber_end < fiber_begin || shell_begin < 0 || shell_end < shell_begin ||
        body_begin < 0 || body_end < body_begin)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_target_ranges: bad ranges");
    fl->rq_f0 = fiber_begin;
    fl->rq_f1 = fiber_end;
    fl->rq_s0 = shell_begin;
    fl->rq_s1 = shell_end;
    fl->rq_b0 = body_begin;
    fl->rq_b1 = body_end;
    fl->use_ranges = true;
    fl->mv_dirty = true;
    fl->ops.invalidate();
    fl->geom_version++;
    return SKB_OK;
}

int skb_flow_last_sym_kernel(const skb_flow *fl, double *ms, int64_t *pairs) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_last_sym_kernel: NULL");
    return fl->fib[1].last_sym_kernel(ms, pairs);
}

int skb_flow_last_stats(const skb_flow *fl, skb_flow_stats *out) {
    if (!fl || !out)
        return set_error(SKB_ERR_INVALID, "skb_flow_last_stats: NULL");
    *out = fl->stats;
    return SKB_OK;
}

} // extern "C"

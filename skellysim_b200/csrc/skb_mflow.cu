// skb_mflow.cu -- ONE process, n GPUs (include/skelly_b200_flow.h): the multi-device shape the reference's "direct
// evaluators need a single rank" rule admits (src/core/system.cpp:618-623).  One group member (skb_flow) per device,
// connected through peer memory; whole fibers, periphery rows and body rows are block-partitioned over the members.
// Every member is driven by its own host thread, so the n launch sequences are issued concurrently.  A client of the
// skb_flow_* API plus the few internals declared in skb_flow.hpp.
#include "skb_flow.hpp"

#include <algorithm>
#include <cmath>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <cstring>
#include <vector>

using namespace skb;

namespace {
class Workers {
  public:
    explicit Workers(int n) : n_(n), task_(n), state_(n, 0), rc_(n, 0), msg_(n) {
        for (int g = 0; g < n; ++g)
            th_.emplace_back([this, g] { loop(g); });
    }
    ~Workers() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_ = true;
        }
        cv_.notify_all();
        for (auto &t : th_)
            t.join();
    }
    // run fn(g) on every worker; returns the first non-zero status (its message becomes this thread's last error)
    int run(const std::function<int(int)> &fn) {
        {
            std::lock_guard<std::mutex> lk(mu_);
            for (int g = 0; g < n_; ++g) {
                task_[g] = fn;
                state_[g] = 1;
            }
        }
        cv_.notify_all();
        std::unique_lock<std::mutex> lk(mu_);
        done_.wait(lk, [this] {
            for (int g = 0; g < n_; ++g)
                if (state_[g] != 0)
                    return false;
            return true;
        });
        for (int g = 0; g < n_; ++g)
            if (rc_[g] != SKB_OK)
                return set_error(rc_[g], "device member %d: %s", g, msg_[g].c_str());
        return SKB_OK;
    }

  private:
    void loop(int g) {
        for (;;) {
            std::function<int(int)> fn;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [this, g] { return stop_ || state_[g] == 1; });
                if (stop_)
                    return;
                fn = task_[g];
            }
            const int rc = fn(g);
            {
                std::lock_guard<std::mutex> lk(mu_);
                rc_[g] = rc;
                msg_[g] = rc == SKB_OK ? "" : last_error();
                state_[g] = 0;
            }
            done_.notify_all();
        }
    }
    int n_;
    std::vector<std::function<int(int)>> task_;
    std::vector<int> state_, rc_;
    std::vector<std::string> msg_;
    std::vector<std::thread> th_;
    std::mutex mu_;
    std::condition_variable cv_, done_;
    bool stop_ = false;
};

} // namespace

struct skb_mflow {
    ~skb_mflow();
    int n = 0;
    std::vector<int> devs;
    std::vector<std::unique_ptr<skb_flow, Destroyer<skb_flow_destroy>>> m;
    std::vector<std::unique_ptr<skb_dense, Destroyer<skb_dense_destroy>>> dn;
    std::unique_ptr<Workers> workers; // declared after m and dn: its threads are joined before any member goes
    // geometry (host copies of what the partition needs)
    long long n_fib = 0, n_shell = 0, n_body = 0;
    int n_fibers = 0, n_bodies = 0;
    std::vector<int> fiber_n;
    std::vector<long long> fiber_off;
    // partition: member g owns fibers [f0[g], f1[g]), periphery rows [s0, s1), body rows [b0, b1)
    std::vector<int> f0, f1;
    std::vector<long long> s0, s1, b0, b1;
    bool part_dirty = true;
    bool has_dense = false, has_minv = false; // skb_mflow_set_dense: stresslet_plus_complementary, M_inv
    bool ops_ready = false;
    std::vector<int> body_n; // node counts of skb_mflow_set_body_operators (the body part of the solution vector)
    long long body_sol = 0;  // ... its size, sum(3 n + 6)
    struct IO {               // per member: the transfers of the host-array call in flight
        Transfers xfer;
        std::vector<DevBuf> stage; // the staging slots of xfer.up, then of xfer.down
        Event e0, e1;
    };
    std::vector<IO> io;
    // skb_mflow_set_gmres: the partition and body node counts it laid the members' local rows out for
    bool gmres_set = false;
    std::vector<long long> gmres_layout;
    skb_flow_stats stats{};
};

// member g of n owns whole fibers [f0, f1) -- cut where the running node count passes g/n of the total
// (fcfd.cpp:102-120 splits by fiber count; by node count balances ragged suspensions as well) -- and equal blocks of
// the periphery and body rows
static void partition_rows(const std::vector<long long> &fiber_off, long long n_shell, long long n_body, int n,
                           std::vector<int> &f0, std::vector<int> &f1, std::vector<long long> &s0,
                           std::vector<long long> &s1, std::vector<long long> &b0, std::vector<long long> &b1) {
    const int n_fibers = (int)fiber_off.size() - 1;
    const long long n_fib = n_fibers > 0 ? fiber_off[(size_t)n_fibers] : 0;
    f0.assign(n, 0), f1.assign(n, 0);
    s0.assign(n, 0), s1.assign(n, 0), b0.assign(n, 0), b1.assign(n, 0);
    int f = 0;
    for (int g = 0; g < n; ++g) {
        f0[g] = f;
        const long long want = n_fib * (g + 1) / n;
        while (f < n_fibers && fiber_off[(size_t)f + 1] <= want)
            ++f;
        if (g == n - 1)
            f = std::max(n_fibers, 0);
        f1[g] = f;
    }
    const long long cs = (n_shell + n - 1) / n, cb = (n_body + n - 1) / n;
    for (int g = 0; g < n; ++g) {
        s0[g] = std::min(n_shell, g * cs);
        s1[g] = std::min(n_shell, (g + 1) * cs);
        b0[g] = std::min(n_body, g * cb);
        b1[g] = std::min(n_body, (g + 1) * cb);
    }
}

static void mflow_partition(skb_mflow *mf) {
    std::vector<long long> off = mf->fiber_off;
    if (off.empty())
        off.push_back(0);
    partition_rows(off, mf->n_shell, mf->n_body, mf->n, mf->f0, mf->f1, mf->s0, mf->s1, mf->b0, mf->b1);
}

// ranges + group wiring, after any change of the geometry's sizes
static int mflow_prepare(skb_mflow *mf) {
    if (!mf->part_dirty)
        return SKB_OK;
    mflow_partition(mf);
    for (int g = 0; g < mf->n; ++g) {
        SKB_TRY(skb_flow_set_target_ranges(mf->m[g].get(), mf->f0[g], mf->f1[g], mf->s0[g], mf->s1[g], mf->b0[g], mf->b1[g]));
        SKB_TRY(skb_flow_group_init(mf->m[g].get(), g, mf->n));
    }
    for (int g = 0; g < mf->n; ++g)
        for (int h = 0; h < mf->n; ++h)
            if (g != h)
                SKB_TRY(skb_flow_group_connect(mf->m[g].get(), h, mf->m[h].get()));
    for (int g = 0; g < mf->n; ++g) // all allocations up front: members may share a device (see skb_flow_group_warmup)
        SKB_TRY(skb_flow_group_warmup(mf->m[g].get()));
    mf->part_dirty = false;
    mf->ops_ready = false;
    return SKB_OK;
}

skb_mflow::~skb_mflow() {
    while (!io.empty()) { // each member's buffers are freed with its device current
        cudaSetDevice(devs[io.size() - 1]);
        io.pop_back();
    }
}

// set(member, a...) on every member in turn, on the calling thread, up to the first that fails
template <class Set, class... A> static int each_member(skb_mflow *mf, const char *who, Set set, A... a) {
    if (!mf)
        return set_error(SKB_ERR_INVALID, "%s: NULL", who);
    for (int g = 0; g < mf->n; ++g)
        SKB_TRY(set(mf->m[g].get(), a...));
    return SKB_OK;
}

extern "C" {

int skb_mflow_create(const int *devices, int n, skb_mflow **out) {
    if (!out || n < 1 || n > kMaxGroup)
        return set_error(SKB_ERR_INVALID, "skb_mflow_create: need 1 <= n <= %d devices", kMaxGroup);
    *out = nullptr;
    std::unique_ptr<skb_mflow> mf(new skb_mflow);
    mf->n = n;
    mf->dn.resize(n);
    for (int g = 0; g < n; ++g) {
        mf->devs.push_back(devices ? devices[g] : g);
        skb_flow *fl = nullptr;
        const int rc = skb_flow_create(mf->devs[g], &fl);
        mf->m.emplace_back(fl);
        SKB_TRY(rc);
        CUDA_TRY(cudaSetDevice(mf->devs[g]));
        mf->io.emplace_back(); // io[g] only once member g exists: ~skb_mflow makes devs[g] current for it
        CUDA_TRY(cudaEventCreate(mf->io[g].e0.out()));
        CUDA_TRY(cudaEventCreate(mf->io[g].e1.out()));
    }
    mf->workers.reset(new Workers(n));
    *out = mf.release();
    return SKB_OK;
}

int skb_mflow_destroy(skb_mflow *mf) {
    if (!mf)
        return SKB_OK;
    mf->workers.reset();
    for (int g = 0; g < mf->n; ++g) {
        cudaSetDevice(mf->devs[g]);
        cudaDeviceSynchronize();
    }
    delete mf;
    return SKB_OK;
}

int skb_mflow_n_devices(const skb_mflow *mf, int *n) {
    if (!mf || !n)
        return set_error(SKB_ERR_INVALID, "skb_mflow_n_devices: NULL");
    *n = mf->n;
    return SKB_OK;
}

int skb_mflow_set_fibers(skb_mflow *mf, const double *r_fib, const int *n_nodes, const double *length, int n_fibers) {
    if (!mf || n_fibers < 0)
        return set_error(SKB_ERR_INVALID, "skb_mflow_set_fibers: bad arguments");
    std::vector<long long> off((size_t)n_fibers + 1, 0);
    for (int f = 0; f < n_fibers; ++f)
        off[(size_t)f + 1] = off[(size_t)f] + (n_nodes ? n_nodes[f] : 0);
    const bool resized = off != mf->fiber_off;
    SKB_TRY(mf->workers->run([&](int g) -> int { return skb_flow_set_fibers(mf->m[g].get(), r_fib, n_nodes, length, n_fibers); }));
    mf->n_fibers = n_fibers;
    mf->n_fib = off[(size_t)n_fibers];
    mf->fiber_off = off;
    mf->fiber_n.assign(n_nodes, n_nodes + n_fibers);
    mf->ops_ready = false;
    if (resized)
        mf->part_dirty = true;
    return SKB_OK;
}

int skb_mflow_set_periphery(skb_mflow *mf, const double *node_pos, const double *node_normal, int64_t n_nodes) {
    if (!mf || n_nodes < 0)
        return set_error(SKB_ERR_INVALID, "skb_mflow_set_periphery: bad arguments");
    SKB_TRY(mf->workers->run([&](int g) -> int { return skb_flow_set_periphery(mf->m[g].get(), node_pos, node_normal, n_nodes); }));
    if (mf->n_shell != n_nodes)
        mf->part_dirty = true;
    mf->n_shell = n_nodes;
    return SKB_OK;
}

int skb_mflow_set_bodies(skb_mflow *mf, const double *node_pos, const double *node_normal, int64_t n_nodes,
                         const double *centers, int n_bodies) {
    if (!mf || n_nodes < 0 || n_bodies < 0)
        return set_error(SKB_ERR_INVALID, "skb_mflow_set_bodies: bad arguments");
    SKB_TRY(mf->workers->run(
        [&](int g) { return skb_flow_set_bodies(mf->m[g].get(), node_pos, node_normal, n_nodes, centers, n_bodies); }));
    if (mf->n_body != n_nodes || mf->n_bodies != n_bodies) // (the window holds 6 partials per body)
        mf->part_dirty = true;
    mf->n_body = n_nodes;
    mf->n_bodies = n_bodies;
    return SKB_OK;
}

int skb_mflow_set_cross(skb_mflow *mf, int mode) {
    SKB_TRY(each_member(mf, "skb_mflow_set_cross", skb_flow_set_cross, mode));
    mf->part_dirty = true; // the members' target lists change: re-run the warm-up
    return SKB_OK;
}

int skb_mflow_set_overlap(skb_mflow *mf, int on) {
    return each_member(mf, "skb_mflow_set_overlap", skb_flow_set_overlap, on);
}

int skb_mflow_set_periphery_shape(skb_mflow *mf, const skb_periphery_shape *shape, const int32_t *fiber_minus_clamped,
                                  const double *body_radius) {
    return each_member(mf, "skb_mflow_set_periphery_shape", skb_flow_set_periphery_shape, shape, fiber_minus_clamped,
                       body_radius);
}

// skb_flow_periphery_interaction of every member into the complete arrays: each member's own fibers, member 0's
// collision test (every member holds the same geometry)
int skb_mflow_periphery_interaction(skb_mflow *mf, double *f_periphery, int32_t *plus_hinged, int32_t *collided) {
    if (!mf)
        return set_error(SKB_ERR_INVALID, "skb_mflow_periphery_interaction: NULL");
    SKB_TRY(mflow_prepare(mf));
    for (int g = 0; g < mf->n; ++g) {
        const int f0 = mf->f0[(size_t)g];
        const long long a = mf->fiber_off[(size_t)f0];
        SKB_TRY(skb_flow_periphery_interaction(mf->m[(size_t)g].get(), f_periphery ? f_periphery + 3 * a : nullptr,
                                               plus_hinged ? plus_hinged + f0 : nullptr, g == 0 ? collided : nullptr));
    }
    return SKB_OK;
}

int skb_mflow_set_self_exclusion(skb_mflow *mf, int fused) {
    return each_member(mf, "skb_mflow_set_self_exclusion", skb_flow_set_self_exclusion, fused);
}

int skb_mflow_partition(skb_mflow *mf, int member, int *fiber_begin, int *fiber_end, int64_t *shell_begin,
                        int64_t *shell_end, int64_t *body_begin, int64_t *body_end) {
    if (!mf || member < 0 || member >= mf->n)
        return set_error(SKB_ERR_INVALID, "skb_mflow_partition: bad member");
    SKB_TRY(mflow_prepare(mf));
    if (fiber_begin) *fiber_begin = mf->f0[member];
    if (fiber_end) *fiber_end = mf->f1[member];
    if (shell_begin) *shell_begin = mf->s0[member];
    if (shell_end) *shell_end = mf->s1[member];
    if (body_begin) *body_begin = mf->b0[member];
    if (body_end) *body_end = mf->b1[member];
    return SKB_OK;
}

// host-only (no GPU needed): the partition skb_mflow uses, for rank-per-GPU hosts that want the same one
int skb_partition_query(const int *n_nodes, int n_fibers, int64_t n_shell, int64_t n_body, int n_members, int member,
                        int64_t *out6) {
    if (n_fibers < 0 || (n_fibers > 0 && !n_nodes) || n_shell < 0 || n_body < 0 || n_members < 1 || member < 0 ||
        member >= n_members || !out6)
        return set_error(SKB_ERR_INVALID, "skb_partition_query: bad arguments");
    std::vector<long long> off((size_t)n_fibers + 1, 0);
    for (int f = 0; f < n_fibers; ++f)
        off[(size_t)f + 1] = off[(size_t)f] + n_nodes[f];
    std::vector<int> f0, f1;
    std::vector<long long> s0, s1, b0, b1;
    partition_rows(off, n_shell, n_body, n_members, f0, f1, s0, s1, b0, b1);
    out6[0] = f0[member], out6[1] = f1[member], out6[2] = s0[member], out6[3] = s1[member], out6[4] = b0[member],
    out6[5] = b1[member];
    return SKB_OK;
}

int skb_mflow_set_fiber_class(skb_mflow *mf, int n_nodes, const double *D_1_0, const double *P_downsample_bc) {
    SKB_TRY(each_member(mf, "skb_mflow_set_fiber_class", skb_flow_set_fiber_class, n_nodes, D_1_0, P_downsample_bc));
    mf->ops_ready = false;
    return SKB_OK;
}

// element offset of fiber f's block in a concatenation of per-fiber (k n) x (4 n) matrices
static long long op_offset(const skb_mflow *mf, int f, int k) {
    long long o = 0;
    for (int i = 0; i < f; ++i)
        o += (long long)k * 4 * mf->fiber_n[(size_t)i] * mf->fiber_n[(size_t)i];
    return o;
}

int skb_mflow_set_fiber_operators(skb_mflow *mf, const double *A, const double *force_operator, const double *xs,
                                  const double *length_prev, const int *plus_bc_velocity) {
    if (!mf)
        return set_error(SKB_ERR_INVALID, "skb_mflow_set_fiber_operators: NULL");
    SKB_TRY(mflow_prepare(mf));
    if (mf->n_fibers > 0 && (!A || !force_operator || !xs || !length_prev || !plus_bc_velocity))
        return set_error(SKB_ERR_INVALID, "skb_mflow_set_fiber_operators: NULL argument");
    SKB_TRY(mf->workers->run([&](int g) -> int {
        const int f0 = mf->f0[g];
        if (mf->f1[g] == f0)
            return skb_flow_set_fiber_operators(mf->m[g].get(), nullptr, nullptr, nullptr, nullptr, nullptr);
        return skb_flow_set_fiber_operators(mf->m[g].get(), A + op_offset(mf, f0, 4), force_operator + op_offset(mf, f0, 3),
                                            xs + 3 * mf->fiber_off[(size_t)f0], length_prev + f0, plus_bc_velocity + f0);
    }));
    mf->ops_ready = true;
    return SKB_OK;
}

int skb_mflow_set_fiber_preconditioner(skb_mflow *mf, const double *A_inv) {
    if (!mf || !mf->ops_ready)
        return set_error(SKB_ERR_INVALID, "skb_mflow_set_fiber_preconditioner: call skb_mflow_set_fiber_operators first");
    return mf->workers->run([&](int g) -> int {
        const int f0 = mf->f0[g];
        return skb_flow_set_fiber_preconditioner(mf->m[g].get(), mf->f1[g] == f0 ? nullptr : A_inv + op_offset(mf, f0, 4));
    });
}

int skb_mflow_set_fiber_class_derivatives(skb_mflow *mf, int n_nodes, const double *D_2_0, const double *D_3_0,
                                          const double *D_4_0) {
    return each_member(mf, "skb_mflow_set_fiber_class_derivatives", skb_flow_set_fiber_class_derivatives, n_nodes,
                       D_2_0, D_3_0, D_4_0);
}

int skb_mflow_build_fiber_operators(skb_mflow *mf, const skb_fiber_params *params, double dt, double eta) {
    if (!mf)
        return set_error(SKB_ERR_INVALID, "skb_mflow_build_fiber_operators: NULL");
    SKB_TRY(mflow_prepare(mf));
    if (mf->n_fibers > 0 && !params)
        return set_error(SKB_ERR_INVALID, "skb_mflow_build_fiber_operators: NULL params");
    SKB_TRY(mf->workers->run([&](int g) -> int {
        return skb_flow_build_fiber_operators(mf->m[g].get(), mf->f1[g] == mf->f0[g] ? nullptr : params + mf->f0[g], dt, eta);
    }));
    mf->ops_ready = true;
    return SKB_OK;
}

int skb_mflow_build_fiber_rhs(skb_mflow *mf, const skb_fiber_params *params, const double *v_growth,
                              const double *force_scale, const double *v_on_fibers, const double *f_external, double dt,
                              double eta, double *rhs) {
    if (!mf)
        return set_error(SKB_ERR_INVALID, "skb_mflow_build_fiber_rhs: NULL");
    SKB_TRY(mflow_prepare(mf));
    if (mf->n_fibers > 0 && (!params || !rhs))
        return set_error(SKB_ERR_INVALID, "skb_mflow_build_fiber_rhs: NULL argument");
    return mf->workers->run([&](int g) -> int {
        const int f0 = mf->f0[g];
        skb_flow *fl = mf->m[g].get();
        if (mf->f1[g] == f0)
            return skb_flow_build_fiber_rhs(fl, nullptr, nullptr, nullptr, nullptr, nullptr, dt, eta, nullptr);
        const long long node = mf->fiber_off[(size_t)f0];
        return skb_flow_build_fiber_rhs(fl, params + f0, v_growth ? v_growth + f0 : nullptr,
                                        force_scale ? force_scale + f0 : nullptr,
                                        v_on_fibers ? v_on_fibers + 3 * node : nullptr,
                                        f_external ? f_external + 3 * node : nullptr, dt, eta, rhs + 4 * node);
    });
}

// the periphery's dense operator, rows block-partitioned like the periphery rows (periphery.cpp:387-417)
int skb_mflow_set_dense(skb_mflow *mf, int op, const double *A_rowmajor, int64_t n_rows, int64_t n_cols) {
    if (!mf || !A_rowmajor || n_rows != 3 * mf->n_shell || n_cols != 3 * mf->n_shell)
        return set_error(SKB_ERR_INVALID, "skb_mflow_set_dense: need the (3 N_s) x (3 N_s) operator of the %lld periphery "
                                          "nodes set before", mf ? mf->n_shell : 0LL);
    SKB_TRY(mflow_prepare(mf));
    SKB_TRY(mf->workers->run([&](int g) -> int {
        if (!mf->dn[g]) {
            skb_dense *dn = nullptr;
            SKB_TRY(skb_dense_create_on(&mf->devs[g], 1, &dn));
            mf->dn[g].reset(dn);
        }
        return skb_dense_set_matrix(mf->dn[g].get(), op, A_rowmajor + (size_t)(3 * mf->s0[g]) * (size_t)n_cols,
                                    3 * (mf->s1[g] - mf->s0[g]), n_cols);
    }));
    if (op == SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY)
        mf->has_dense = true;
    if (op == SKB_DENSE_M_INV)
        mf->has_minv = true;
    return SKB_OK;
}

static int mflow_collect_stats(skb_mflow *mf) {
    double dev_ms = 0;
    long long pairs = 0;
    int launches = 0;
    for (int g = 0; g < mf->n; ++g) {
        float ms = 0;
        cudaSetDevice(mf->devs[g]);
        if (cudaEventElapsedTime(&ms, mf->io[g].e0, mf->io[g].e1) == cudaSuccess)
            dev_ms = std::max(dev_ms, (double)ms);
        else
            (void)cudaGetLastError();
        skb_flow_stats st{};
        skb_flow_last_stats(mf->m[g].get(), &st);
        pairs += st.n_pairs;
        launches += st.launches;
        int missing = -1;
        SKB_TRY(skb_flow_group_error(mf->m[g].get(), &missing));
        if (missing >= 0)
            return set_error(SKB_ERR_STATE, "device member %d timed out waiting for member %d (a peer failed or never "
                                            "issued the matching call)", g, missing);
    }
    mf->stats.device_ms = dev_ms;
    mf->stats.total_ms = dev_ms;
    mf->stats.n_pairs = pairs;
    mf->stats.launches = launches;
    return SKB_OK;
}

} // extern "C"

// rows of member g: fiber nodes [a, a + n_fw), n_fibers whole fibers, n_sw periphery rows, n_bw body rows
struct MemberRows {
    long long a, n_fw, n_sw, n_bw;
    int n_fibers;
};
static MemberRows member_rows(const skb_mflow *mf, int g) {
    const long long a = mf->fiber_off.empty() ? 0 : mf->fiber_off[(size_t)mf->f0[g]],
                    b = mf->fiber_off.empty() ? 0 : mf->fiber_off[(size_t)mf->f1[g]];
    return MemberRows{a, b - a, mf->s1[g] - mf->s0[g], mf->b1[g] - mf->b0[g], mf->f1[g] - mf->f0[g]};
}

// On the calling thread, before any worker starts: member g's transfers of the call, describe(g), and the staging slots
// they need, sized there -- cudaMalloc / cudaFree may synchronise the whole device and must not run while a peer on the
// same device sits in a flag wait.  A slot holds at least 8 bytes, so a member call gets a device pointer for an empty
// array too.  The background streamer's buffers take their size here as well.
template <class Describe> static int mflow_stage(skb_mflow *mf, Describe describe) {
    for (int g = 0; g < mf->n; ++g) {
        CUDA_TRY(cudaSetDevice(mf->devs[g]));
        skb_mflow::IO &io = mf->io[g];
        io.xfer = describe(g);
        SKB_TRY(stage_slots(io.stage, io.xfer));
        const long long n_sw = mf->s1[g] - mf->s0[g];
        if (mf->has_dense && n_sw > 0 && mf->m[g]->bg.enabled) // the background streamer's, if it is on
            SKB_TRY(overlap_buffers(mf->m[g].get(), 3 * n_sw));
    }
    return SKB_OK;
}

// On member g's worker: the uploads mflow_stage described, call(stream, transfers) between the member's timing events,
// then the downloads and, if the call has any, the wait for them.  Allocates nothing.
template <class Call> static int member_call(skb_mflow *mf, int g, Call call) {
    const skb_mflow::IO &io = mf->io[(size_t)g];
    CUDA_TRY(cudaSetDevice(mf->devs[(size_t)g]));
    const cudaStream_t st = mf->m[(size_t)g]->stream;
    SKB_TRY(issue(io.xfer.up, true, st));
    CUDA_TRY(cudaEventRecord(io.e0, st));
    SKB_TRY(call(st, io.xfer));
    CUDA_TRY(cudaEventRecord(io.e1, st));
    SKB_TRY(issue(io.xfer.down, false, st));
    if (!io.xfer.down.empty())
        CUDA_TRY(cudaStreamSynchronize(st));
    return SKB_OK;
}

extern "C" {

// v_all over [fibers | periphery | bodies] like skb_flow_matvec; complete host arrays in and out
int skb_mflow_matvec(skb_mflow *mf, const double *fib_forces, const double *shell_density, const double *body_densities,
                     const double *body_forces_torques, double eta, double *v_all) {
    if (!mf || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "skb_mflow_matvec: bad arguments");
    const long long nf = mf->n_fib, ns = mf->n_shell, nb = mf->n_body;
    if ((nf > 0 && !fib_forces) || (ns > 0 && !shell_density) || (nb > 0 && !body_densities) ||
        (mf->n_bodies > 0 && !body_forces_torques) || (nf + ns + nb > 0 && !v_all))
        return set_error(SKB_ERR_INVALID, "skb_mflow_matvec: NULL input for a non-empty class");
    SKB_TRY(mflow_prepare(mf));
    std::vector<double> f, t;
    if (mf->n_bodies > 0)
        split_forces_torques(body_forces_torques, mf->n_bodies, f, t);
    const long long n_ft = (long long)f.size();
    SKB_TRY(mflow_stage(mf, [&](int g) -> Transfers {
        const MemberRows r = member_rows(mf, g);
        return {{up(fib_forces, {{3 * r.a, 0, 3 * r.n_fw}}), up(shell_density, {{3 * mf->s0[g], 0, 3 * r.n_sw}}),
                 up(body_densities, {{0, 0, 3 * nb}}), up(f.data(), {{0, 0, n_ft}}), up(t.data(), {{0, 0, n_ft}})},
                {down(v_all, {{3 * r.a, 0, 3 * r.n_fw},
                              {3 * (nf + mf->s0[g]), 3 * r.n_fw, 3 * r.n_sw},
                              {3 * (nf + ns + mf->b0[g]), 3 * (r.n_fw + r.n_sw), 3 * r.n_bw}})}};
    }));
    SKB_TRY(mf->workers->run([&](int g) -> int {
        return member_call(mf, g, [&](cudaStream_t st, const Transfers &io) {
            return skb_flow_matvec_device(mf->m[g].get(), io.up[0].dev, io.up[1].dev, io.up[2].dev, io.up[3].dev,
                                          io.up[4].dev, eta, io.down[0].dev, st);
        });
    }));
    return mflow_collect_stats(mf);
}

// System::apply_matvec (system.cpp:269-324) over n devices: complete host arrays in and out.  out_shell = res_shell
// when skb_mflow_set_dense(SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY) was called, else v_shell.
int skb_mflow_apply_matvec(skb_mflow *mf, const double *x_fibers, const double *x_shell, const double *body_densities,
                           const double *body_forces_torques, const double *fiber_link_conditions, double eta,
                           double *res_fibers, double *out_shell, double *v_bodies) {
    if (!mf || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "skb_mflow_apply_matvec: bad arguments");
    if (!mf->ops_ready && mf->n_fibers > 0) // no fibers: the empty operator set, uploaded or not
        return set_error(SKB_ERR_STATE, "skb_mflow_apply_matvec: call skb_mflow_set_fiber_operators first");
    const long long nf = mf->n_fib, ns = mf->n_shell, nb = mf->n_body;
    if ((nf > 0 && (!x_fibers || !res_fibers)) || (ns > 0 && (!x_shell || !out_shell)) ||
        (nb > 0 && (!body_densities || !v_bodies)) || (mf->n_bodies > 0 && !body_forces_torques))
        return set_error(SKB_ERR_INVALID, "skb_mflow_apply_matvec: NULL argument for a non-empty class");
    SKB_TRY(mflow_prepare(mf));
    std::vector<double> f, t;
    if (mf->n_bodies > 0)
        split_forces_torques(body_forces_torques, mf->n_bodies, f, t);
    const long long n_ft = (long long)f.size();
    SKB_TRY(mflow_stage(mf, [&](int g) -> Transfers {
        const MemberRows r = member_rows(mf, g);
        const long long s0 = mf->s0[g], b0 = mf->b0[g];
        return {{up(x_fibers, {{4 * r.a, 0, 4 * r.n_fw}}), up(x_shell, {{3 * s0, 0, 3 * r.n_sw}}),
                 up(body_densities, {{0, 0, 3 * nb}}), up(f.data(), {{0, 0, n_ft}}), up(t.data(), {{0, 0, n_ft}}),
                 up(fiber_link_conditions, {{7LL * mf->f0[g], 0, 7LL * r.n_fibers}})},
                {down(res_fibers, {{4 * r.a, 0, 4 * r.n_fw}}), down(out_shell, {{3 * s0, 0, 3 * r.n_sw}}),
                 down(v_bodies, {{3 * b0, 0, 3 * r.n_bw}})}};
    }));
    SKB_TRY(mf->workers->run([&](int g) -> int {
        const bool links = fiber_link_conditions && mf->f1[g] > mf->f0[g];
        return member_call(mf, g, [&](cudaStream_t st, const Transfers &io) {
            return skb_flow_apply_matvec_device(mf->m[g].get(), mf->has_dense ? mf->dn[g].get() : nullptr,
                                                io.up[0].dev, io.up[1].dev, io.up[2].dev, io.up[3].dev, io.up[4].dev,
                                                links ? io.up[5].dev : nullptr, eta, io.down[0].dev, io.down[1].dev,
                                                io.down[2].dev, st);
        });
    }));
    return mflow_collect_stats(mf);
}

} // extern "C"

// ---- the whole-vector calls [fibers | shell | bodies] over n devices: every member runs its skb_flow_group_* call ----
// Row ownership: member g owns its fibers' rows, its periphery rows and, of the body part, the 3 rows of each body node
// in [b0, b1) and the six rows [U; w] of every body whose first node lies in [b0, b1) (skellysim_b200.distributed
// .system_rows).  A member's local vector holds those rows in ascending order.

static long long mflow_solution_size(const skb_mflow *mf) {
    return 4 * mf->n_fib + 3 * mf->n_shell + (mf->n_bodies > 0 ? mf->body_sol : 0);
}

// member g's slice of a per-fiber array of all fibers, k entries per fiber (NULL stays NULL, and so does the slice of a
// member without fibers)
template <class T> static T *own_slice(const skb_mflow *mf, int g, T *all, int k = 1) {
    return all && mf->f1[(size_t)g] > mf->f0[(size_t)g] ? all + (size_t)k * mf->f0[(size_t)g] : nullptr;
}

// member g's rows of a whole vector in its local order [fiber rows | shell rows | body pieces], one run per non-empty
// piece
static std::vector<Run> member_local(const skb_mflow *mf, int g) {
    const MemberRows r = member_rows(mf, g);
    const long long body = 4 * mf->n_fib + 3 * mf->n_shell, at = 4 * r.n_fw + 3 * r.n_sw;
    std::vector<RowPiece> pieces;
    if (mf->n_bodies > 0)
        body_row_pieces(mf->body_n.data(), (int)mf->body_n.size(), mf->b0[(size_t)g], mf->b1[(size_t)g], pieces);
    std::vector<Run> runs;
    if (r.n_fw)
        runs.push_back({4 * r.a, 0, 4 * r.n_fw});
    if (r.n_sw)
        runs.push_back({4 * mf->n_fib + 3 * mf->s0[(size_t)g], 4 * r.n_fw, 3 * r.n_sw});
    for (const RowPiece &p : pieces)
        runs.push_back({body + p.body, at + p.local, p.len});
    return runs;
}

// On the calling thread, before any worker starts: every member whose rows are not laid out for its current ranges (a
// new partition re-runs skb_flow_group_init) lays them out for the recorded bodies
static int mflow_local_rows(skb_mflow *mf, const char *who) {
    if (mf->n_bodies > 0 && (int)mf->body_n.size() != mf->n_bodies)
        return set_error(SKB_ERR_INVALID, "%s: call skb_mflow_set_body_operators first", who);
    for (int g = 0; g < mf->n; ++g) {
        skb_flow *fl = mf->m[(size_t)g].get();
        CUDA_TRY(cudaSetDevice(fl->dev));
        SKB_TRY(prepare_matvec_targets(fl));
        if (fl->grp.member() && !fl->grp.rows_for(group_ranges(fl)))
            SKB_TRY(flow_member_lay_out_rows(fl, who, mf->body_n.data(), mf->n_bodies));
    }
    return SKB_OK;
}

// the bodies' node counts the members' local rows are laid out by
static void mflow_set_body_n(skb_mflow *mf, const int *n_nodes, int n_bodies) {
    mf->body_n.assign(n_nodes, n_nodes + n_bodies);
    mf->body_sol = 0;
    for (int n : mf->body_n)
        mf->body_sol += 3LL * n + 6;
}

// the link checks of every fiber (a member checks its own fibers only), leaving the links the flow holds as they are
static int check_fiber_links(skb_flow *fl, const int *body, const double *site, const double *rigidity) {
    CUDA_TRY(cudaSetDevice(fl->dev));
    return fl->bodies.set_links(all_fibers(fl), fl->ops, fl->n_bodies, fl->h_centers.data(), body, site, rigidity,
                                fl->stream, true);
}

extern "C" {

int skb_mflow_set_body_operators(skb_mflow *mf, const int *n_nodes, int n_bodies, const double *node_weights,
                                 const double *ex, const double *ey, const double *ez, const double *A_inv) {
    const char *who = "skb_mflow_set_body_operators";
    if (!mf)
        return set_error(SKB_ERR_INVALID, "%s: NULL", who);
    if (n_bodies != mf->n_bodies)
        return set_error(SKB_ERR_INVALID, "%s: %d bodies, skb_mflow_set_bodies has %d", who, n_bodies, mf->n_bodies);
    if (n_bodies > 0 && (!n_nodes || !node_weights || !ex || !ey || !ez))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    SKB_TRY(mflow_prepare(mf));
    // every member checks the same complete arrays first, so all of them refuse or none does
    SKB_TRY(mf->workers->run([&](int g) -> int {
        return skb_flow_group_set_body_operators(mf->m[g].get(), n_nodes, n_bodies, node_weights, ex, ey, ez, A_inv);
    }));
    mflow_set_body_n(mf, n_nodes, n_bodies);
    return SKB_OK;
}

int skb_mflow_set_body_frames(skb_mflow *mf, const int *n_nodes, int n_bodies, const double *node_pos_ref,
                              const double *node_normal_ref, const double *node_weights, const double *ex0,
                              const double *ey0, const double *ez0, const double *A_inv0) {
    const char *who = "skb_mflow_set_body_frames";
    if (!mf)
        return set_error(SKB_ERR_INVALID, "%s: NULL", who);
    if (n_bodies != mf->n_bodies)
        return set_error(SKB_ERR_INVALID, "%s: %d bodies, skb_mflow_set_bodies has %d", who, n_bodies, mf->n_bodies);
    if (n_bodies > 0 && (!n_nodes || !node_pos_ref || !node_normal_ref || !node_weights || !ex0 || !ey0 || !ez0))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    SKB_TRY(mflow_prepare(mf));
    // every member checks the same complete arrays first, so all of them refuse or none does
    SKB_TRY(mf->workers->run([&](int g) -> int {
        return skb_flow_group_set_body_frames(mf->m[g].get(), n_nodes, n_bodies, node_pos_ref, node_normal_ref,
                                              node_weights, ex0, ey0, ez0, A_inv0);
    }));
    mflow_set_body_n(mf, n_nodes, n_bodies); // the layout every placement keeps
    return SKB_OK;
}

int skb_mflow_place_bodies(skb_mflow *mf, const double *centers, const double *orientations) {
    if (!mf)
        return set_error(SKB_ERR_INVALID, "skb_mflow_place_bodies: NULL");
    SKB_TRY(mflow_prepare(mf));
    std::vector<double> R;
    for (int g = 0; g < mf->n; ++g) // every member's refusals before any member places
        SKB_TRY(placement_args(mf->m[g].get(), "skb_mflow_place_bodies", centers, orientations, R));
    return mf->workers->run([&](int g) -> int { return skb_flow_group_place_bodies(mf->m[g].get(), centers, orientations); });
}

int skb_mflow_set_fiber_links(skb_mflow *mf, const int *body, const double *site, const double *bending_rigidity) {
    const char *who = "skb_mflow_set_fiber_links";
    if (!mf)
        return set_error(SKB_ERR_INVALID, "%s: NULL", who);
    if (body && mf->n_fibers > 0 && (!site || !bending_rigidity))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    SKB_TRY(mflow_prepare(mf));
    SKB_TRY(check_fiber_links(mf->m[0].get(), body, site, bending_rigidity)); // before any member replaces its links
    return mf->workers->run([&](int g) -> int {
        return skb_flow_group_set_fiber_links(mf->m[g].get(), own_slice(mf, g, body), own_slice(mf, g, site, 3),
                                              own_slice(mf, g, bending_rigidity));
    });
}

// the refusals of both system calls, before any launch; then every member's rows are laid out
static int mflow_system_args(skb_mflow *mf, const char *who, bool precondition, bool args) {
    if (!mf)
        return set_error(SKB_ERR_INVALID, "%s: NULL", who);
    SKB_TRY(mflow_prepare(mf)); // (a new partition drops the fiber operators)
    if (!mf->ops_ready && mf->n_fibers > 0) // no fibers: the empty operator set, uploaded or not
        return set_error(SKB_ERR_STATE, "%s: call skb_mflow_set_fiber_operators first", who);
    for (int g = 0; g < mf->n; ++g)
        SKB_TRY(system_ready(mf->m[g].get(), who, kMflowCalls, precondition));
    const int op = precondition ? SKB_DENSE_M_INV : SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY;
    const char *op_name = precondition ? "SKB_DENSE_M_INV" : "SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY";
    if (mf->n_shell > 0 && !(precondition ? mf->has_minv : mf->has_dense))
        return set_error(SKB_ERR_INVALID, "%s: the periphery needs its dense operator (skb_mflow_set_dense with %s)",
                         who, op_name);
    // each member's row block must fit the periphery as it is now (skb_mflow_set_periphery may have changed its size)
    for (int g = 0; g < mf->n && mf->n_shell > 0; ++g) {
        const long long n_sw = mf->s1[g] - mf->s0[g];
        int64_t rows = -1, cols = -1;
        if (n_sw > 0 && mf->dn[g])
            SKB_TRY(skb_dense_shape(mf->dn[g].get(), op, &rows, &cols));
        if (n_sw > 0 && (rows != 3 * n_sw || cols != 3 * mf->n_shell))
            return set_error(SKB_ERR_INVALID, "%s: device member %d holds a %lld x %lld block of %s, need its %lld rows "
                                              "x %lld of the %lld periphery nodes (call skb_mflow_set_dense again after "
                                              "skb_mflow_set_periphery)", who, g, (long long)rows, (long long)cols,
                             op_name, 3 * n_sw, 3 * mf->n_shell, mf->n_shell);
    }
    if (!args)
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    return mflow_local_rows(mf, who);
}

// member g's rows of the whole host vector `in` up into its local vector, its local result down into the whole `out`
static Transfers member_vector(const skb_mflow *mf, int g, const double *in, double *out, double *d_in = nullptr,
                               double *d_out = nullptr) {
    const std::vector<Run> rows = member_local(mf, g);
    return {{up(in, rows, d_in)}, {down(out, rows, d_out)}};
}

// member g's uploads of the external forces: its fibers' rows of f_external, the bodies' complete forces and torques
static std::vector<Transfer> external_forces(const skb_mflow *mf, int g, const double *f_external,
                                             const std::vector<double> &f, const std::vector<double> &t) {
    const MemberRows r = member_rows(mf, g);
    const long long n_ft = (long long)f.size();
    return {up(f_external, {{3 * r.a, 0, 3 * r.n_fw}}), up(f.data(), {{0, 0, n_ft}}), up(t.data(), {{0, 0, n_ft}})};
}

// System::apply_matvec (system.cpp:269-324) over n devices on the whole solution vector
int skb_mflow_apply_system_matvec(skb_mflow *mf, const double *x, double eta, double *res) {
    const char *who = "skb_mflow_apply_system_matvec";
    SKB_TRY(mflow_system_args(mf, who, false, (x && res) || (mf && mflow_solution_size(mf) == 0)));
    if (!(eta > 0))
        return set_error(SKB_ERR_INVALID, "%s: eta = %g", who, eta);
    if (mflow_solution_size(mf) == 0)
        return SKB_OK;
    SKB_TRY(mflow_stage(mf, [&](int g) { return member_vector(mf, g, x, res); }));
    SKB_TRY(mf->workers->run([&](int g) -> int {
        skb_dense *dn = mf->has_dense ? mf->dn[g].get() : nullptr;
        return member_call(mf, g, [&](cudaStream_t st, const Transfers &io) {
            return skb_flow_group_apply_system_matvec_device(mf->m[g].get(), dn, io.up[0].dev, eta, io.down[0].dev, st);
        });
    }));
    return mflow_collect_stats(mf);
}

// System::apply_preconditioner (system.cpp:248-262) over n devices
int skb_mflow_apply_system_preconditioner(skb_mflow *mf, const double *x, double *y) {
    const char *who = "skb_mflow_apply_system_preconditioner";
    SKB_TRY(mflow_system_args(mf, who, true, (x && y) || (mf && mflow_solution_size(mf) == 0)));
    if (mflow_solution_size(mf) == 0)
        return SKB_OK;
    SKB_TRY(mflow_stage(mf, [&](int g) { return member_vector(mf, g, x, y); }));
    SKB_TRY(mf->workers->run([&](int g) -> int {
        return member_call(mf, g, [&](cudaStream_t st, const Transfers &io) {
            return skb_flow_group_apply_system_preconditioner_device(mf->m[g].get(), mf->dn[g].get(), io.up[0].dev,
                                                                     io.down[0].dev, st);
        });
    }));
    return mflow_collect_stats(mf);
}

// System::prep_state_for_solver's RHS (system.cpp:398-458) over n devices: every member forms its own rows of the
// whole vector.  The flow is the group's matvec flow (strengths pushed to every window, the members' partial sums pulled
// together); the bodies' external F_T are complete on every member and enter the body flow as they are.
int skb_mflow_build_system_rhs(skb_mflow *mf, const skb_fiber_params *params, const double *v_growth,
                               const double *force_scale, const double *f_external, const double *body_forces_torques,
                               double dt, double eta, double *rhs) {
    const char *who = "skb_mflow_build_system_rhs";
    if (!mf)
        return set_error(SKB_ERR_INVALID, "%s: NULL", who);
    if (!(dt > 0) || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "%s: dt = %g, eta = %g (both must be > 0)", who, dt, eta);
    SKB_TRY(mflow_prepare(mf));
    auto finite = [](const double *a, size_t n) {
        for (size_t i = 0; i < n; ++i)
            if (!std::isfinite(a[i]))
                return false;
        return true;
    };
    if ((f_external && !finite(f_external, (size_t)mf->n_fib * 3)) ||
        (body_forces_torques && !finite(body_forces_torques, (size_t)mf->n_bodies * 6)))
        return set_error(SKB_ERR_INVALID, "%s: a non-finite external force or torque", who);
    if (mf->n_fibers > 0 && !params)
        return set_error(SKB_ERR_INVALID, "%s: NULL params", who);
    // every member's checks and buffers, on this thread, before any member launches (a refusal after a peer had pushed
    // its strengths would leave that peer waiting on a flag)
    for (int g = 0; g < mf->n; ++g)
        SKB_TRY(flow_member_rhs_prepare(mf->m[g].get(), params, v_growth, force_scale, dt, eta));
    const long long n = mflow_solution_size(mf);
    if (n > 0 && !rhs)
        return set_error(SKB_ERR_INVALID, "%s: NULL rhs", who);
    if (n == 0)
        return SKB_OK;
    std::vector<double> f, t;
    if (body_forces_torques && mf->n_bodies > 0)
        split_forces_torques(body_forces_torques, mf->n_bodies, f, t);
    SKB_TRY(mflow_local_rows(mf, who));
    SKB_TRY(mflow_stage(mf, [&](int g) -> Transfers {
        return {external_forces(mf, g, f_external, f, t), {down(rhs, member_local(mf, g))}};
    }));
    SKB_TRY(mf->workers->run([&](int g) -> int {
        return member_call(mf, g, [&](cudaStream_t st, const Transfers &io) {
            return skb_flow_group_build_system_rhs_device(
                mf->m[g].get(), own_slice(mf, g, params), own_slice(mf, g, v_growth), own_slice(mf, g, force_scale),
                f_external ? io.up[0].dev : nullptr, f.empty() ? nullptr : io.up[1].dev,
                t.empty() ? nullptr : io.up[2].dev, dt, eta, io.down[0].dev, st);
        });
    }));
    return mflow_collect_stats(mf);
}

// the analytic sources of velocity_at_targets and of the system RHS, on every member
int skb_mflow_set_point_sources(skb_mflow *mf, const double *positions, const double *forces, const double *torques,
                                int n_points) {
    return each_member(mf, "skb_mflow_set_point_sources", skb_flow_set_point_sources, positions, forces, torques,
                       n_points);
}

int skb_mflow_set_background(skb_mflow *mf, const int *components, const double *scale_factor,
                             const double *uniform) {
    return each_member(mf, "skb_mflow_set_background", skb_flow_set_background, components, scale_factor, uniform);
}

// System::velocity_at_targets (system.cpp:330-384) over n devices: the targets are block-partitioned, every device
// holds all sources
int skb_mflow_velocity_at_targets(skb_mflow *mf, const double *r_trg, int64_t n_trg, const double *fib_forces,
                                  const double *shell_density, const double *body_densities,
                                  const double *body_forces_torques, double eta, double *vel) {
    if (!mf || n_trg < 0 || (n_trg > 0 && (!r_trg || !vel)) || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "skb_mflow_velocity_at_targets: bad arguments");
    const long long chunk = (n_trg + mf->n - 1) / mf->n;
    SKB_TRY(mf->workers->run([&](int g) -> int {
        const long long b = std::min<long long>(n_trg, g * chunk), e = std::min<long long>(n_trg, (g + 1) * chunk);
        if (e <= b)
            return (int)SKB_OK;
        return skb_flow_velocity_at_targets(mf->m[g].get(), r_trg + 3 * b, e - b, fib_forces, shell_density, body_densities,
                                            body_forces_torques, eta, vel + 3 * b);
    }));
    double dev_ms = 0;
    long long pairs = 0;
    int launches = 0;
    for (int g = 0; g < mf->n; ++g) {
        skb_flow_stats st{};
        skb_flow_last_stats(mf->m[g].get(), &st);
        dev_ms = std::max(dev_ms, st.device_ms);
        pairs += st.n_pairs;
        launches += st.launches;
    }
    mf->stats.device_ms = mf->stats.total_ms = dev_ms;
    mf->stats.n_pairs = pairs;
    mf->stats.launches = launches;
    return SKB_OK;
}

int skb_mflow_last_stats(const skb_mflow *mf, skb_flow_stats *out) {
    if (!mf || !out)
        return set_error(SKB_ERR_INVALID, "skb_mflow_last_stats: NULL");
    *out = mf->stats;
    return SKB_OK;
}

} // extern "C"

// ---- the solve (skb_mflow_set_gmres / _solve_system): every member runs skb_flow_group_solve_system_device ----------
static std::vector<long long> gmres_layout(const skb_mflow *mf) {
    std::vector<long long> v;
    for (int g = 0; g < mf->n; ++g)
        v.insert(v.end(), {(long long)mf->f0[g], (long long)mf->f1[g], mf->s0[g], mf->s1[g], mf->b0[g], mf->b1[g]});
    v.insert(v.end(), mf->body_n.begin(), mf->body_n.end());
    return v;
}

// the members' rows must still be those skb_mflow_set_gmres laid out
static int mflow_gmres_current(const skb_mflow *mf, const char *who) {
    if (mf->gmres_set && mf->gmres_layout == gmres_layout(mf))
        return SKB_OK;
    return set_error(SKB_ERR_INVALID, "%s: call skb_mflow_set_gmres after the partition or the bodies' node counts "
                                      "changed", who);
}

extern "C" {

int skb_mflow_set_gmres(skb_mflow *mf, int num_blocks) {
    const char *who = "skb_mflow_set_gmres";
    if (!mf)
        return set_error(SKB_ERR_INVALID, "%s: NULL", who);
    if (num_blocks < 1 || num_blocks > kMaxKrylov)
        return set_error(SKB_ERR_INVALID, "%s: num_blocks = %d (must be in [1, %d])", who, num_blocks, kMaxKrylov);
    SKB_TRY(mflow_prepare(mf));
    SKB_TRY(mflow_local_rows(mf, who));
    mf->gmres_set = false;
    SKB_TRY(mf->workers->run([&](int g) -> int { return skb_flow_set_gmres(mf->m[(size_t)g].get(), num_blocks); }));
    mf->gmres_layout = gmres_layout(mf);
    mf->gmres_set = true;
    return SKB_OK;
}

int skb_mflow_solve_system(skb_mflow *mf, const double *rhs, double eta, double tol, int num_blocks, int max_iters,
                           double *x, skb_solve_info *info, double *history) {
    const char *who = "skb_mflow_solve_system";
    const bool empty = mf && mflow_solution_size(mf) == 0;
    // every member's refusals before any device starts: a member that went on alone would wait on its peers' flags
    SKB_TRY(mflow_system_args(mf, who, false, (rhs && x) || empty));
    SKB_TRY(mflow_system_args(mf, who, true, (rhs && x) || empty));
    if (!(eta > 0))
        return set_error(SKB_ERR_INVALID, "%s: eta = %g", who, eta);
    SKB_TRY(solve_scalar_args(who, tol, num_blocks, max_iters));
    if (!info)
        return set_error(SKB_ERR_INVALID, "%s: NULL info", who);
    if (empty) {
        std::memset(info, 0, sizeof(*info));
        info->converged = 1;
        return SKB_OK;
    }
    SKB_TRY(mflow_gmres_current(mf, who));
    for (int g = 0; g < mf->n; ++g) {
        skb_flow *fl = mf->m[(size_t)g].get();
        long long n = 0;
        std::array<long long, 6> key;
        SKB_TRY(flow_gmres_size(fl, who, &n, &key));
        if (!fl->kry.sized_for(n, key) || num_blocks > fl->kry.blocks())
            return set_error(SKB_ERR_INVALID, "%s: num_blocks = %d, skb_mflow_set_gmres sized device member %d for %d",
                             who, num_blocks, g, fl->kry.blocks());
    }
    std::vector<skb_solve_info> infos((size_t)mf->n);
    std::vector<std::vector<double>> hist((size_t)mf->n, std::vector<double>(history ? (size_t)max_iters + 1 : 0));
    SKB_TRY(mflow_stage(mf, [&](int g) {
        const Krylov &kry = mf->m[(size_t)g]->kry;
        return member_vector(mf, g, rhs, x, kry.stage_b(), kry.stage_x());
    }));
    SKB_TRY(mf->workers->run([&](int g) -> int {
        skb_dense *dn = mf->dn[(size_t)g].get();
        return member_call(mf, g, [&](cudaStream_t st, const Transfers &io) {
            return skb_flow_group_solve_system_device(mf->m[(size_t)g].get(), dn, dn, io.up[0].dev, eta, tol,
                                                      num_blocks, max_iters, io.down[0].dev, &infos[(size_t)g],
                                                      history ? hist[(size_t)g].data() : nullptr, st);
        });
    }));
    for (int g = 1; g < mf->n; ++g) // the all-reduce leaves every member the same scalars
        if (std::memcmp(&infos[(size_t)g], &infos[0], sizeof(skb_solve_info)) != 0 || hist[(size_t)g] != hist[0])
            return set_error(SKB_ERR_STATE, "%s: device member %d ended its solve unlike member 0", who, g);
    *info = infos[0];
    if (history)
        std::memcpy(history, hist[0].data(), (size_t)(info->iterations + 1) * 8);
    return mflow_collect_stats(mf);
}

// System::step over the devices: skb_flow_group_step_device's run on every member's thread, after every member's
// refusals on this one.  The members all-gather the body rows and the new fiber geometry through their group windows,
// so every member takes the same decision and installs the same complete geometry
int skb_mflow_step(skb_mflow *mf, const skb_fiber_params *params, const double *v_growth, const double *force_scale,
                   const double *f_external, const double *body_forces_torques, const int *fiber_body,
                   const double *site_ref, double dt, double eta, double tol, int num_blocks, int max_iters, double *x,
                   double *tension, skb_step_info *info) {
    const char *who = "skb_mflow_step";
    // ---- every member's refusals, before any member launches: a member that refused on its own thread would leave
    // its peers waiting on a flag ----
    if (!mf)
        return set_error(SKB_ERR_INVALID, "%s: NULL", who);
    const int nb = mf->n_bodies;
    SKB_TRY(step_scalar_args(who, info, dt, eta, tol, num_blocks, max_iters));
    SKB_TRY(step_fiber_args(who, params, fiber_body, site_ref, 0, mf->n_fibers, nb));
    SKB_TRY(step_host_inputs(who, f_external, mf->n_fib, body_forces_torques, nb));
    SKB_TRY(mflow_prepare(mf));
    if (mf->n_shell > 0 && (!mf->has_dense || !mf->has_minv))
        return set_error(SKB_ERR_INVALID, "%s: the periphery needs both dense operators (skb_mflow_set_dense)", who);
    if (mflow_solution_size(mf) == 0) { // the empty system: nothing moves
        std::memset(info, 0, sizeof(*info));
        info->worst_fiber = -1;
        info->solve.converged = 1;
        return SKB_OK;
    }
    SKB_TRY(mflow_gmres_current(mf, who));
    std::vector<StepArgs> args((size_t)mf->n);
    std::vector<StepCall> calls((size_t)mf->n);
    for (int g = 0; g < mf->n; ++g) {
        skb_flow *fl = mf->m[(size_t)g].get();
        args[(size_t)g] = StepArgs{own_slice(mf, g, params),     own_slice(mf, g, v_growth),
                                   own_slice(mf, g, force_scale), own_slice(mf, g, fiber_body),
                                   own_slice(mf, g, site_ref, 3), dt, eta, tol, num_blocks, max_iters};
        skb_dense *dn = mf->dn[(size_t)g].get();
        SKB_TRY(group_step_checks(fl, dn, dn, args[(size_t)g], info, who, calls[(size_t)g]));
        // (also the RHS's buffers at their size and its tables uploaded, as every skb_mflow RHS does first)
        SKB_TRY(flow_member_rhs_prepare(fl, params, v_growth, force_scale, dt, eta));
    }
    std::vector<double> f, t;
    if (body_forces_torques && nb > 0)
        split_forces_torques(body_forces_torques, nb, f, t);
    SKB_TRY(mflow_stage(mf, [&](int g) { return Transfers{external_forces(mf, g, f_external, f, t), {}}; }));

    // ---- every member's step; its local rows of the solution and its own tensions into the complete host arrays ----
    std::vector<skb_step_info> infos((size_t)mf->n);
    const int rc = mf->workers->run([&](int g) -> int {
        std::vector<double> loc(x ? (size_t)calls[(size_t)g].n : 0);
        int rc_g = SKB_OK;
        SKB_TRY(member_call(mf, g, [&](cudaStream_t st, const Transfers &io) {
            skb_dense *dn = mf->dn[(size_t)g].get();
            rc_g = group_step_run(mf->m[(size_t)g].get(), dn, dn, args[(size_t)g], calls[(size_t)g],
                                  f_external ? io.up[0].dev : nullptr, f.empty() ? nullptr : io.up[1].dev,
                                  t.empty() ? nullptr : io.up[2].dev, x ? loc.data() : nullptr,
                                  tension ? tension + member_rows(mf, g).a : nullptr, &infos[(size_t)g], who, st);
            return rc_g == SKB_ERR_STATE ? SKB_OK : rc_g; // (SKB_ERR_STATE: not installed, the outputs are there)
        }));
        if (x)
            for (const Run &p : member_local(mf, g))
                std::memcpy(x + p.whole, loc.data() + p.at, (size_t)p.len * 8);
        return rc_g;
    });
    mf->ops_ready = rc == SKB_ERR_STATE; // built by the step; an installed step set new fibers, which drops them
    if (rc != SKB_OK && rc != SKB_ERR_STATE)
        return rc;
    for (int g = 1; g < mf->n; ++g) // the members decided from the same complete arrays
        if (std::memcmp(&infos[(size_t)g], &infos[0], sizeof(skb_step_info)) != 0)
            return set_error(SKB_ERR_STATE, "%s: device member %d ended its step unlike member 0", who, g);
    *info = infos[0];
    SKB_TRY(mflow_collect_stats(mf));
    return rc; // (SKB_ERR_STATE keeps the message of the member that reported it)
}

// every member holds the same geometry: member 0's
int skb_mflow_get_fibers(skb_mflow *mf, double *r_fib) {
    if (!mf)
        return set_error(SKB_ERR_INVALID, "skb_mflow_get_fibers: NULL");
    return skb_flow_get_fibers(mf->m[0].get(), r_fib);
}

int skb_mflow_get_placement(skb_mflow *mf, double *centers, double *orientations) {
    if (!mf)
        return set_error(SKB_ERR_INVALID, "skb_mflow_get_placement: NULL");
    return skb_flow_get_placement(mf->m[0].get(), centers, orientations);
}

} // extern "C"

// skb_flow.hpp -- the flow (include/skelly_b200_flow.h) and what the translation units built on it share:
// skb_flow.cu (its lifetime, geometry, knobs and statistics), skb_matvec.cu (its flows and matvec orchestration),
// skb_system.cu (the whole-system calls and the fiber operators' entry points), skb_listener.cu (the listener's
// requests), skb_solve.cu, skb_step.cu, skb_periphery.cu and skb_mflow.cu.  Free functions in namespace skb that take
// the flow.
#pragma once
#include "skb_internal.hpp"
#include "../../include/skelly_b200_flow.h"
#include "../../include/skelly_b200_dense.h"

#include <array>
#include <cstring>
#include <memory>
#include <vector>

namespace skb {
// The copies of one host-array call (the flow's and skb_mflow's): each Run moves len doubles between the caller's array
// at `whole` and the device array at `at`
struct Run {
    long long whole, at, len;
};
struct Transfer {
    double *host;          // the caller's array (only read by an upload); NULL: nothing to copy
    double *dev;           // a device array the callee owns, or the staging slot stage_slots gives it
    std::vector<Run> runs;
};
struct Transfers {
    std::vector<Transfer> up, down; // before the call, after it
};
inline Transfer up(const double *h, std::vector<Run> runs, double *dev = nullptr) {
    return Transfer{const_cast<double *>(h), dev, std::move(runs)};
}
inline Transfer down(double *h, std::vector<Run> runs, double *dev = nullptr) {
    return Transfer{h, dev, std::move(runs)};
}
// the whole array of n doubles
inline Transfer up(const double *h, long long n) { return up(h, {{0, 0, n}}); }
inline Transfer down(double *h, long long n) { return down(h, {{0, 0, n}}); }
// Every transfer of x without a device array gets one of `slots` (the slots of x.up, then those of x.down), grown to
// 8 bytes beyond the end of its runs, so that a call gets a device pointer for an empty array too.  Slots only grow;
// a transfer that has a device array keeps it.  May allocate: skb_mflow stages on the calling thread
int stage_slots(std::vector<DevBuf> &slots, Transfers &x);
// the runs of `list` issued on st: x.up host to device (upload true), x.down device to host
int issue(const std::vector<Transfer> &list, bool upload, cudaStream_t st);

struct TargetCache {
    std::vector<double> host;
    bool valid = false;
    unsigned long long version = 0; // bumped by every upload: part of the CUDA-graph key (a replay bakes in whether
                                    // the symmetric path -- targets start with the sources -- was taken)
    bool same(const double *r, long long n) const {
        return valid && (long long)host.size() == 3 * n && (n == 0 || std::memcmp(host.data(), r, (size_t)n * 24) == 0);
    }
    void store(const double *r, long long n) {
        host.assign(r, r + 3 * n);
        valid = true;
        ++version;
    }
    // another call has put other targets into the evaluator: the next call with host targets uploads them again
    void invalidate() {
        valid = false;
        ++version;
    }
};

// the step's device buffers: per fiber its item and error, per fiber node its new position and tension, the external
// forces and torques of the RHS; and a pinned host copy of skb_flow_group_step_device's device inputs (3 per fiber
// node + 6 per body)
// for their finiteness check.  Sized by skb_flow_set_gmres (the step itself allocates none of them)
struct StepBuffers {
    DevBuf items, r_new, tension, err, fext, force, torque;
    PinnedHost check;
    int size(int n_fibers, long long n_fib, int n_bodies);
    bool sized_for(int n_fibers, long long n_fib, int n_bodies) const {
        return n_fibers_ == n_fibers && n_fib_ == n_fib && n_bodies_ == n_bodies;
    }

  private:
    int n_fibers_ = -1, n_bodies_ = -1;
    long long n_fib_ = -1;
    size_t check_cap_ = 0; // doubles of `check`
};

// The periphery's shape (skb_flow_set_periphery_shape) and what the step derives from it on the device: the
// fiber-periphery repulsion, the plus-end binding and the collision test (skb_periphery.cu, periphery_kernels.cuh).
// Holds the per-fiber and per-body tables of the call, and the buffers of one pass sized for the fibers it was set or
// sized for (a group step allocates nothing).  The caller has made the flow's device current
class PeripheryShape {
  public:
    // checked first: a refusal leaves the earlier shape.  kind NONE clears it
    int set(const ::skb_periphery_shape *shape, const int *minus_clamped, const double *body_radius, int n_fibers,
            long long n_fib, int n_bodies, long long n_shell, cudaStream_t st);
    bool active() const { return active_; }
    // the pass's buffers for n_fib nodes (skb_flow_set_gmres); a no-op without a shape
    int size(long long n_fib);
    // the per-fiber and per-body tables were set for this many fibers and bodies (only set() changes them)
    bool counts_fit(int n_fibers, int n_bodies) const { return n_fibers == n_fibers_ && n_bodies == n_bodies_; }
    // the pass's buffers hold n_fib nodes (set() or size())
    bool nodes_fit(long long n_fib) const { return n_fib <= cap_nodes_; }
    // is_minus_clamped() of fibers [f0, f0 + nf) from a step's params: the collision test skips their node 0 then
    void note_clamped(int f0, int nf, const ::skb_fiber_params *params);
    // the same flags of ALL fibers as the group step all-gathered them (1.0 / 0.0 per fiber)
    void note_clamped_all(const std::vector<double> &flags);
    // the per-fiber tables of n_old fibers carried to a new set of n_fibers fibers (skb_flow_dynamic_instability):
    // fiber j takes the flags of fiber origin[j], 0 where origin[j] < 0; the pass's buffers sized for n_fib nodes.  A
    // no-op without a shape, or when the tables were set for another fiber count (a step then refuses, as before)
    int carry(const int *origin, int n_old, int n_fibers, long long n_fib, cudaStream_t st);
    // minus_clamped of params (fibers [f0, f0 + nf)) uploaded on st into the device table the group step's kernel
    // reads (clamp_table(), indexed by fiber among ALL fibers), without noting them
    int upload_clamped(int f0, int nf, const ::skb_fiber_params *params, cudaStream_t st);
    const int *clamp_table() const { return (const int *)collide_skip_.ptr; }
    // one launch over the fibers [f0, f1) of offsets d_off and positions d_r_fib (and, with bodies, the n_bodies
    // centres d_centers): the repulsion of their nodes into force() (with_force), their flags into flags() (host,
    // f1 - f0 entries, then the bodies' flag); returns once the flags are on the host
    int run(const double *d_r_fib, const long long *d_off, int f0, int f1, bool with_force, const double *d_centers,
            int n_bodies, cudaStream_t st, int *launches);
    const double *force() const { return (const double *)force_.ptr; }
    const int *flags() const { return (const int *)h_flags_.get(); }
    // d_out = d_in + force() over n doubles (d_in NULL: force() alone)
    int add_force(const double *d_in, double *d_out, long long n, cudaStream_t st, int *launches) const;

  private:
    bool active_ = false;
    ::skb_periphery_shape s_{};
    int n_fibers_ = -1, n_bodies_ = -1;
    long long cap_nodes_ = -1;
    size_t flag_cap_ = 0; // ints of h_flags_
    std::vector<int> h_clamped_; // the collision test's node-0 skip per fiber
    std::vector<int> h_force_skip_; // fiber_minus_clamped of the call (the repulsion's node-0 skip)
    DevBuf force_skip_, collide_skip_, radius_, force_, flags_;
    PinnedHost h_flags_;
};

// The listener's frame (skb_flow_set_listener_frame) and the device state of its requests (skb_listener.cu,
// listener_kernels.cuh): the strengths and the bodies' rigid motions of one solution, valid while the flow's
// geom_version is the one they were set at; the lines' state and output, grow-only
class Listener {
  public:
    int set_frame(skb_flow *fl, const double *fib_forces, const double *shell_density, const double *body_densities,
                  const double *body_forces_torques, const double *body_velocities, const int32_t *body_kind,
                  const double *body_radii, double eta);
    // skb_flow_set_listener_state(_device): the frame of the installed geometry and a step's solution.  device: x and
    // tension are device pointers whose writes the caller ordered on st
    int set_state(skb_flow *fl, const ::skb_fiber_params *params, double dt, double eta, const double *tension,
                  const double *x, const int32_t *body_kind, const double *body_radii, int periphery_interaction,
                  bool device, cudaStream_t st);
    int velocity(skb_flow *fl, const double *r_trg, long long n_trg, double *vel);
    // skb_flow_listener_gradient: d u_i / d x_j (9 per target) and the pressure (1 per target)
    int gradient(skb_flow *fl, const double *r_trg, long long n_trg, double *grad, double *pressure);
    int lines(skb_flow *fl, int kind, const double *x0, int n_lines, const ::skb_line_request *req, double *x,
              double *t, double *val, int32_t *n_points, int32_t *status);

  private:
    // the frame's buffers are written on the flow's stream: wait for them, then the frame is current
    int commit(skb_flow *fl, int n_interior, double eta);
    // the refusal of a request without a current frame
    int current(const skb_flow *fl, const char *who) const;
    // System::velocity_at_targets of the frame at the n_trg device targets d_trg into d_v, on the flow's stream
    int eval(skb_flow *fl, const double *d_trg, long long n_trg, double *d_v);
    // the arbitrary-target evaluators take the n_trg device targets d_trg (the plain kernel only), and the host-target
    // calls are told to upload their own again
    int take_targets(skb_flow *fl, const double *d_trg, long long n_trg);

    bool set_ = false;
    unsigned long long version_ = 0;
    double eta_ = 0;
    int n_interior_ = 0; // bodies with an interior test
    DevBuf ff_, sd_, bd_, f_, t_, rigid_; // strengths; per body [kind, r0, r1, r2, cx, cy, cz, U, omega]
    DevBuf xf_, sb_, ten_; // set_state: the packed [x; y; z; T] per fiber; the host form's shell and body blocks, tension
    DevBuf trg_, vel_;                     // targets and velocities of one evaluation
    DevBuf g10_, grad_, p_;                // gradient: the sums (10 per target), then the gradient and the pressure
    // lines: state (SoA) and per-line output; slot -> line map and the active count of the last compaction
    DevBuf st_x_, st_t_, st_dt_, st_k_, st_int_, out_x_, out_t_, out_val_, slots_, n_act_;
    PinnedHost h_n_act_;
};
// The bodies' nucleation sites (skb_flow_set_nucleation_sites) and the buffers of skb_flow_dynamic_instability
// (skb_dynamic.cu, dynamic_kernels.cuh)
struct DynamicInstability {
    std::vector<int> site_count;     // per body
    std::vector<long long> site_off; // first flat site of every body (n_bodies + 1)
    std::vector<double> site_ref;    // 3 per site, body frame, bodies concatenated
    bool sites_set = false;
    DevBuf d_site_ref, fib, len_new, counts, src, dst_off, picks, frames, r_new, len_out;
    PinnedHost h_counts; // DiCounts, then the keep bytes, then the occupancy bytes
    size_t h_cap = 0;    // bytes of h_counts
};
} // namespace skb

struct skb_flow {
    int dev = 0;
    skb::Stream stream;
    skb::Event ev0, ev1, evt0, evt1;
    // geometry
    long long n_fib = 0, n_shell = 0, n_body = 0;
    int n_fibers = 0, n_bodies = 0, max_fiber_nodes = 0;
    skb::DevBuf fiber_offset, fiber_length, r_fib, r_shell, r_body, centers;
    std::vector<double> h_r_fib, h_r_shell, h_r_body; // host copies to assemble the matvec target lists
    // evaluators: [0] arbitrary targets, [1] matvec target lists
    skb::Evaluator fib[2], shell[2], body[2];
    skb::TargetCache tc_fib, tc_shell, tc_body;
    bool mv_dirty = true;
    int cross_mode = -1;    // fiber <-> periphery cross kernel in the matvec: -1 auto, 0 off, 1 on whenever applicable
    // how matvec_core evaluates, decided by prepare_matvec_targets
    struct MatvecPlan {
        bool grouped = false; // group member: the strengths come packed from the group window (push), not the caller
        // producer of the fiber rows: the plain kernel; the symmetric kernel's complete rows (whole system on this
        // device, cross kernel); or this member's symmetric partial sums, pulled together from all members' windows
        enum FiberRows { kPlain, kSymComplete, kSymPartial } fib_rows = kPlain;
        bool cross = false;   // fiber <-> periphery pairs through the cross kernel
    } plan;
    skb::CrossState cross;
    bool self_excl = false; // matvec: skip intra-fiber pairs in the kernels instead of compute-then-subtract (N3, opt-in)
    long long win_begin = 0, win_end = -1; // target window of the matvec in [fibers|shell|bodies] rows; -1 = all
    bool use_ranges = false;               // skb_flow_set_target_ranges instead of a contiguous window
    long long rq_f0 = 0, rq_f1 = 0, rq_s0 = 0, rq_s1 = 0, rq_b0 = 0, rq_b1 = 0; // requested (fiber indices, rows)
    // resolved pieces of the matvec target list: fiber rows [fa,fb), shell rows [sa,sb), body rows [ba,bb);
    // the output has n_win = (fb-fa)+(sb-sa)+(bb-ba) rows in that order
    long long fa = 0, fb = 0, sa = 0, sb = 0, ba = 0, bb = 0, n_win = 0;
    cudaStream_t cur = nullptr;            // stream of the call in flight (own stream or the caller's)
    int n_points = 0;
    skb::DevBuf pt_pos, pt_force, pt_torque;
    bool has_background = false;
    // CUDA-graph replay of the launch-bound small-size calls (BASELINE C1, listener / streamline path)
    struct GraphSlot {
        skb::GraphExec exec;
        unsigned long long key = 0, seen = 0;
        int launches = 0;
        long long pairs = 0;
        void reset() {
            exec.reset();
            key = seen = 0;
        }
    } g_matvec, g_vat;
    unsigned long long geom_version = 1;
    bool graphs_enabled = true;
    skb::PinnedHost h_stage; // pinned staging: the graph's memcpy nodes need fixed host addresses
    size_t h_stage_cap = 0;
    int bg_comp[3] = {0, 1, 2};
    double bg_scale[3] = {0, 0, 0}, bg_uniform[3] = {0, 0, 0};
    std::vector<int> h_fiber_n;         // nodes of every fiber
    std::vector<long long> h_fiber_off; // first node of every fiber (n_fibers + 1)
    skb::FiberOps ops; // per-fiber dense operators of the fibers whose rows are in the target list (skb_fiber.cu)
    skb::BodyOps bodies; // the bodies' operators and the fiber-body links of the whole-vector operator (skb_body.cu)
    std::vector<double> h_centers; // body centres (set_fiber_links measures the nucleation sites from them)
    std::vector<double> h_fiber_len; // length_ of every fiber (the time step installs its new positions with them)
    std::vector<double> h_orient;    // the quaternions of the last skb_flow_place_bodies (4 per body) ...
    bool placed = false;             // ... valid until skb_flow_set_bodies changes the bodies otherwise
    skb::StepBuffers stepbuf;             // the buffers of skb_flow_step (skb_step.cu)
    skb::PeripheryShape shape;            // skb_flow_set_periphery_shape (skb_periphery.cu)
    skb::Listener listener;               // skb_flow_set_listener_frame and its requests (skb_listener.cu)
    skb::DynamicInstability dyn;          // skb_flow_set_nucleation_sites, skb_flow_dynamic_instability
    std::vector<int> step_hinged;         // plus_hinged each fiber was built with by the last installed step
    skb::Group grp; // multi-GPU group membership: one member per GPU, exchange through peer memory (skb_group.cu)
    // a member's whole-vector matvec in flight: matvec_core exchanges the bodies' partial link forces through the
    // window and the body flow reads their totals from ft_sum ([F | L], 6 per body)
    bool ft_exchange = false;
    skb::DevBuf ft_sum;
    // a rank-per-GPU member's whole-vector matvec has begun the epoch (and exchanged its body rows in it): matvec_core
    // runs its protocol in that epoch instead of beginning one
    bool grp_open = false;
    skb::DevBuf sys_rb; // a member's body output in the whole body layout (skb_flow_group_*), compacted to its own rows
    // Periphery::matvec's dense operator beside the pair kernels (stream_kernels.cuh): forked onto bg_stream once its
    // input (the complete x_shell) is there, joined before res_shell is assembled
    struct Overlap {
        bool enabled = true;       // skb_flow_set_overlap
        skb::Stream stream;
        skb::Event fork, join;
        skb::DevBuf y;                  // A x of the own periphery rows
        skb_dense *dn = nullptr;   // pending background product of the call in flight (nullptr: none)
        bool launched = false;
    } bg;
    // The device cores' workspace, like sys_rb and ft_sum above: they read and write it, and no transfer of a
    // host-array call ever targets it.  vel: v_all of apply_matvec_core and the system RHS; fw: the fibers' force of apply_matvec_core; tmp: the
    // periphery rows of matvec_core; tmp_b: the system matvec's v_bodies; scratch_u: group mode's landing zone of
    // Evaluator::eval's default output (never read)
    skb::DevBuf vel, fw, tmp, tmp_b, scratch_u;
    skb::DevBuf zeros; // the system RHS: the zero densities (and absent forces) its flow takes, n_zeros doubles
    long long n_zeros = 0;
    // the staging slots of the host-array calls (host_call): their inputs and outputs on the device
    std::vector<skb::DevBuf> slots;
    skb::Krylov kry; // the workspace of skb_flow_solve_system (skb_solve.cu)
    skb_flow_stats stats{};
    int launches = 0;
    long long pairs = 0;
};

namespace skb {
// every fiber of the flow
inline OwnFibers all_fibers(const skb_flow *fl) {
    return OwnFibers{0, fl->n_fibers, fl->h_fiber_n.data(), fl->h_fiber_off.data(), (const double *)fl->r_fib.ptr,
                     (const double *)fl->fiber_length.ptr, fl->stream};
}

// ---- skb_flow.cu ----
// The fibers whose operators are resident: those whose rows are in this flow's target list -- all of them, or the
// rank's own fibers under skb_flow_set_target_ranges / an aligned skb_flow_set_target_window.
int own_fibers(skb_flow *fl, const char *who, OwnFibers &own);
int upload(skb_flow *fl, DevBuf &buf, const double *h, size_t n_doubles);
int download(skb_flow *fl, double *h, const DevBuf &buf, size_t n_doubles);
void begin_stats(skb_flow *fl);
int finish_stats(skb_flow *fl);
// the device-pointer entry points run asynchronously on the caller's stream: no timings
int device_stats(skb_flow *fl);

// frame of the host-pointer entry points on fl->stream: device_ms spans the device work, total_ms also the uploads
// before it and the downloads after it; returns once the downloads have landed
template <class Up, class Work, class Down> int host_frame(skb_flow *fl, Up up, Work work, Down down) {
    fl->cur = fl->stream;
    CUDA_TRY(cudaEventRecord(fl->evt0, fl->stream));
    SKB_TRY(up());
    CUDA_TRY(cudaEventRecord(fl->ev0, fl->stream));
    SKB_TRY(work());
    CUDA_TRY(cudaEventRecord(fl->ev1, fl->stream));
    SKB_TRY(down());
    CUDA_TRY(cudaEventRecord(fl->evt1, fl->stream));
    return finish_stats(fl);
}
// the step of host_frame that has nothing to do
inline int nothing() { return SKB_OK; }
// Frame of the flow's host-array calls: x staged into the flow's slots (stage_slots), then in host_frame x's uploads
// and before() (a call's own uploads, such as FiberOps::rhs's tables), work(x), x's downloads; returns once the
// downloads have landed
template <class Work, class Before = int (*)()>
int host_call(skb_flow *fl, Transfers &x, Work work, Before before = nothing) {
    SKB_TRY(stage_slots(fl->slots, x));
    return host_frame(
        fl,
        [&]() -> int {
            SKB_TRY(issue(x.up, true, fl->stream));
            return before();
        },
        [&] { return work((const Transfers &)x); }, [&] { return issue(x.down, false, fl->stream); });
}
// frame of the device-pointer entry points: work on the caller's stream, then the statistics of no timing
template <class Work> int device_frame(skb_flow *fl, void *stream, Work work) {
    fl->cur = (cudaStream_t)stream;
    SKB_TRY(work());
    return device_stats(fl);
}

// ---- skb_matvec.cu ----
// resolve the target window / ranges into fiber, shell and body pieces and (re)build the matvec target lists
int prepare_matvec_targets(skb_flow *fl);
// skb_flow_set_fibers' device part, once the fibers' offsets, lengths and positions are on the device: the self term's
// shared-memory limit for fibers of fl->max_fiber_nodes nodes, and the trapezoid weights of both fiber source sets
int install_fiber_sources(skb_flow *fl);
// the background streamer's buffers for n_rows own periphery rows
int overlap_buffers(skb_flow *fl, long long n_rows);
// device-side matvec flow on fl->cur, as fl->plan says: d_ff / d_sd are the strengths of the own fibers / periphery
// rows (all of them without a group), body inputs are complete; d_v = [own fiber rows | own shell rows | own body rows]
// of v_all
int matvec_core(skb_flow *fl, const double *d_ff, const double *d_sd, const double *d_bd, const double *d_f,
                const double *d_t, double eta, double *d_v);
// System::apply_matvec (system.cpp:298-319) on fl->cur, everything device resident.  Inputs are the OWN slices of a
// group member (all of them without a group): d_x 4 per own fiber node, d_xs 3 per own periphery row, body inputs
// complete, d_link 7 per own fiber or NULL.  Outputs: d_res_fib 4 per own node, d_out_shell 3 per own periphery row
// (res_shell when dn != NULL, else v_shell), d_v_bodies 3 per own body row; any of them may be NULL when empty.
int apply_matvec_core(skb_flow *fl, skb_dense *dn, const double *d_x, const double *d_xs, const double *d_bd,
                      const double *d_f, const double *d_t, const double *d_link, double eta, double *d_res_fib,
                      double *d_out_shell, double *d_v_bodies);
// + psc.flow(r_trg, eta, time) + bs.flow(r_trg, eta) (system.cpp:358-359, 445-446) on st: the point sources of
// skb_flow_set_point_sources and the background flow of skb_flow_set_background at the n_trg targets d_trg, added to
// the rows of d_v in this order: Oseen contraction, rotlet, background
int add_sources(skb_flow *fl, const double *d_trg, long long n_trg, double eta, double *d_v, cudaStream_t st);
// System::velocity_at_targets without its body-interior replacement (system.cpp:355-359) on fl->cur: the fibers'
// flow (no self subtraction), the bodies', the periphery's and add_sources at the n_trg device targets d_trg, which
// the arbitrary-target evaluators fib[0], shell[0] and body[0] hold as their targets.  Strengths as the evaluators take
// them: d_ff 3 per fiber node, d_sd 3 per periphery node, d_bd 3 per body node, d_f and d_t 3 per body
int velocity_dev(skb_flow *fl, const double *d_trg, long long n_trg, const double *d_ff, const double *d_sd,
                 const double *d_bd, const double *d_f, const double *d_t, double eta, double *d_v);
// The velocity gradient and the pressure of the same sum (and the same evaluators' targets) into d_g, 10 per target:
// d u_i / d x_j at 10 t + 3 i + j, and the pressure over eta at 10 t + 9 (the pair kernels' post-scale carries 1 / eta
// for all ten outputs).  Overwrites d_g
int gradient_dev(skb_flow *fl, const double *d_trg, long long n_trg, const double *d_ff, const double *d_sd,
                 const double *d_bd, const double *d_f, const double *d_t, double eta, double *d_g);
int load_source_kernels(); // the kernels of add_sources and gradient_dev, loaded now

// ---- skb_system.cu: the whole-system calls ----
// the whole solution vector's size (of every member alike)
long long solution_size(const skb_flow *fl);
// a rank-per-GPU member: the resolved target ranges its set-up sized its buffers for (prepare_matvec_targets has run),
// and the size of its local vector
Group::Ranges group_ranges(const skb_flow *fl);
long long group_local_size(const skb_flow *fl);

// The family of calls whose set-up calls a refusal names: `setup` prefixes the calls that set the bodies' operators,
// frames and links, `geometry` those that set the fibers and bodies
struct Calls {
    const char *setup, *geometry;
};
constexpr Calls kFlowCalls{"skb_flow_", "skb_flow_"}, kMflowCalls{"skb_mflow_", "skb_mflow_"},
    kGroupCalls{"skb_flow_group_", "skb_flow_"};
// What the system calls need besides the dense operator: an error naming `who` unless it is there.  The fiber
// operators (with their inverse for the preconditioner), the body operators (with their inverse for the preconditioner)
// and, for the matvec, the fiber links.  step: the step, which builds the fiber operators and sets the links itself but
// places the bodies from their frames (precondition: the frames' inverse)
int system_ready(skb_flow *fl, const char *who, const Calls &calls, bool precondition, bool step = false);
// dn holds this flow's rows of the periphery operator of a system call (matvec: stresslet_plus_complementary;
// precondition: M_inv): on the flow's device, 3 (sb - sa) rows x 3 n_shell
int dense_rows(skb_flow *fl, skb_dense *dn, const char *who, bool precondition);
// an error naming `who` unless the flow's target list is the whole system; `hint` ends the message
int whole_targets(skb_flow *fl, const char *who, const char *hint);
// The checks of the system operator of a single-device flow (matvec: stresslet_plus_complementary in dn; precondition:
// M_inv and the inverses), all before any launch; then the flow's device is current and its target list resolved.
int system_args(skb_flow *fl, skb_dense *dn, const char *who, bool precondition, bool args);
// the same for a group member's local-vector calls
int group_system_args(skb_flow *fl, skb_dense *dn, const char *who, bool precondition);

// the size and key skb_flow_set_gmres sizes for (a member: its local rows, which need its rows laid out)
int flow_gmres_size(skb_flow *fl, const char *who, long long *n, std::array<long long, 6> *key);
// a group member (else nothing): lays out its own body rows for bodies of n_nodes and sizes every buffer its
// local-vector calls use (what skb_flow_group_set_body_operators / _set_body_frames do besides the operators)
int flow_member_lay_out_rows(skb_flow *fl, const char *who, const int *n_nodes, int n_bodies);

// R (row-major) of a unit quaternion (w, x, y, z): the formula of Eigen's QuaternionBase::toRotationMatrix
void quaternion_rotation(const double *q, double *R);
// the refusals of a placement, before any state changes, with the rotations R (9 per body) it places at
int placement_args(skb_flow *fl, const char *who, const double *centers, const double *orientations,
                   std::vector<double> &R);

// skb_mflow_build_system_rhs on one member, on the calling thread before any member launches: the refusals (the
// member's fibers and bodies; params / v_growth / force_scale of ALL fibers), the upload of the fiber block's per-fiber
// tables, and every buffer and kernel the RHS uses
int flow_member_rhs_prepare(skb_flow *fl, const ::skb_fiber_params *params, const double *v_growth,
                            const double *force_scale, double dt, double eta);

// ---- skb_solve.cu ----
// the refusals of a solve's tol, num_blocks and max_iters (each caller checks its own eta)
int solve_scalar_args(const char *who, double tol, int num_blocks, int max_iters);

// ---- the time step (skb_step.cu), which skb_mflow_step drives on every member ----
// the per-fiber arguments of a step (of the fibers it steps: a group member's own) and its scalars
struct StepArgs {
    const ::skb_fiber_params *params;
    const double *v_growth, *force_scale;
    const int *fiber_body;
    const double *site_ref;
    double dt, eta, tol;
    int num_blocks, max_iters;
};
// what a step's refusals leave for its run: the fibers it steps, their items, bending rigidity and current nucleation
// sites, and the (local) solution size
struct StepCall {
    OwnFibers own;
    std::vector<StepItem> items;
    std::vector<double> rigidity, sites;
    long long n = 0;
    // with a periphery shape: the own fibers' params with plus_hinged from the binding (empty: the caller's params)
    std::vector<::skb_fiber_params> hinged;
    const ::skb_fiber_params *params(const StepArgs &a) const { return hinged.empty() ? a.params : hinged.data(); }
};

// ---- the periphery's shape in the step (skb_periphery.cu) ----
// an error naming `who` unless a periphery shape is set and fits the flow as it is
int periphery_ready(const skb_flow *fl, const char *who);
// d_ff += the repulsion of every fiber node at the current geometry (fc.periphery_force, system.cpp:340-341) on st;
// refuses a non-finite repulsion.  After periphery_ready
int periphery_add_repulsion(skb_flow *fl, const char *who, double *d_ff, cudaStream_t st, int *launches);
// with a shape: the pass over the own fibers at the current geometry (the repulsion kept for
// periphery_add_force, c.hinged filled); refuses a non-finite repulsion and a shape not set or sized for the flow.
// Changes nothing the step's refusal would have to undo.  Without a shape: nothing
int periphery_before_step(skb_flow *fl, const char *who, const StepArgs &a, StepCall &c);
// d_out = d_f_external + the repulsion of the m own nodes of periphery_before_step (d_f_external NULL: the repulsion)
int periphery_add_force(skb_flow *fl, const double *d_f_external, long long m, double *d_out, cudaStream_t st,
                        int *launches);
// System::check_collision of the flow's current geometry, ALL fibers and bodies (0 without a shape)
int periphery_collided(skb_flow *fl, int *collided, cudaStream_t st, int *launches);
// the refusals of the step's host arguments: the scalars; params, fiber_body and site_ref of nf fibers (the first is
// fiber f0) against nb bodies; the external forces of n_fib fiber nodes and the forces and torques of nb bodies finite
int step_scalar_args(const char *who, const ::skb_step_info *info, double dt, double eta, double tol, int num_blocks,
                     int max_iters);
int step_fiber_args(const char *who, const ::skb_fiber_params *params, const int *fiber_body, const double *site_ref,
                    int f0, int nf, int nb);
int step_host_inputs(const char *who, const double *f_external, long long n_fib, const double *body_forces_torques,
                     int nb);
// skb_flow_group_step_device in two halves (on a flow that is no member, such as a one-device skb_mflow's, those of
// skb_flow_step).  group_step_checks: every refusal except the device inputs' finiteness, before any launch, with the
// arguments of the member's own fibers.  group_step_run: the step itself, which meets the member's peers at flag
// waits -- every member's checks must have passed first.  Inputs on the device as the
// public call takes them; x_local / tension (host or device memory, NULL: not wanted) receive the member's local rows
// of the solution and its own fibers' tensions, also when the step is not installed (SKB_ERR_STATE)
int group_step_checks(skb_flow *fl, skb_dense *dn_spc, skb_dense *dn_minv, const StepArgs &a, ::skb_step_info *info,
                      const char *who, StepCall &c);
int group_step_run(skb_flow *fl, skb_dense *dn_spc, skb_dense *dn_minv, const StepArgs &a, StepCall &c,
                   const double *d_f_external, const double *d_body_forces, const double *d_body_torques,
                   double *x_local, double *tension, ::skb_step_info *info, const char *who, cudaStream_t st);
} // namespace skb

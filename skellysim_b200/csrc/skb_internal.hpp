// skb_internal.hpp -- declarations shared by the translation units of libskelly_b200.so
#pragma once
#include "../../include/skelly_b200.h"

#include <array>
#include <cuda_runtime.h>
#include <functional>
#include <map>
#include <stddef.h>
#include <type_traits>
#include <utility>
#include <vector>

struct skb_fiber_params;
struct skb_solve_info;

namespace skb {

struct DeviceInfo {
    int dev = 0;
    int num_sms = 0;
    // [kind][T index: 1,2,4,8] resident CTAs / SM; the gradient kinds (2, 3) run at kGradT only
    int occupancy[4][4] = {{1, 1, 1, 1}, {1, 1, 1, 1}, {1, 1, 1, 1}, {1, 1, 1, 1}};
};

struct LaunchPlan {
    int T = 4;               // targets per consumer thread
    int n_splits = 1;        // source splits (gridDim.y)
    int tiles_per_split = 1; // source tiles per split
    unsigned grid_x = 1;     // target tiles
};

// Device memory with one owner.  The destructor frees it; the device it lives on must be current then.
struct DevBuf {
    void *ptr = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(DevBuf &&o) noexcept { *this = std::move(o); }
    DevBuf &operator=(DevBuf &&o) noexcept { // o takes the old buffer and frees it
        std::swap(ptr, o.ptr);
        std::swap(cap, o.cap);
        return *this;
    }
    ~DevBuf() {
        if (ptr)
            cudaFree(ptr);
    }
    int ensure(size_t bytes); // grow-only; contents are NOT preserved
    // ensure(bytes), then the host bytes h copied in on st (asynchronously); nothing at all for 0 bytes
    int upload(const void *h, size_t bytes, cudaStream_t st);
};
static_assert(!std::is_copy_constructible<DevBuf>::value && !std::is_copy_assignable<DevBuf>::value,
              "a copy would free the buffer twice");

// One CUDA handle (stream, event, graph exec, pinned or IPC-mapped pointer) and the call that releases it.  Converts to
// the raw handle, so launches and API calls take it unchanged; out() hands its address to the call that creates it.
template <class H, auto Release> class Owned {
    H h_ = nullptr;

  public:
    Owned() = default;
    Owned(Owned &&o) noexcept : h_(o.h_) { o.h_ = nullptr; }
    Owned &operator=(Owned &&o) noexcept {
        std::swap(h_, o.h_);
        return *this;
    }
    ~Owned() { reset(); }
    operator H() const { return h_; }
    H get() const { return h_; }
    H *out() {
        reset();
        return &h_;
    }
    void reset() {
        if (h_)
            Release(h_);
        h_ = nullptr;
    }
};
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using Event = Owned<cudaEvent_t, cudaEventDestroy>;
using GraphExec = Owned<cudaGraphExec_t, cudaGraphExecDestroy>;
using PinnedHost = Owned<double *, cudaFreeHost>;
using DevPtr = Owned<void *, cudaFree>;              // exact-size allocation (DevBuf rounds up)
using IpcPtr = Owned<void *, cudaIpcCloseMemHandle>; // a peer's memory mapped into this process

// unique_ptr deleter of a library object: its C API destroy function
template <auto Destroy> struct Destroyer {
    template <class T> void operator()(T *p) const { Destroy(p); }
};

int set_error(int code, const char *fmt, ...) __attribute__((format(printf, 2, 3)));
// return from the enclosing function with the error of a failed CUDA call / library call
#define CUDA_TRY(expr)                                                                                                \
    do {                                                                                                              \
        cudaError_t _e = (expr);                                                                                      \
        if (_e != cudaSuccess)                                                                                        \
            return ::skb::set_error(SKB_ERR_CUDA, "%s failed at %s:%d: %s", #expr, __FILE__, __LINE__,                \
                                    cudaGetErrorString(_e));                                                          \
    } while (0)
#define SKB_TRY(expr)                                                                                                 \
    do {                                                                                                              \
        int _rc = (expr);                                                                                             \
        if (_rc != SKB_OK)                                                                                            \
            return _rc;                                                                                               \
    } while (0)
const char *last_error();
void count_launch(int n);
long long launch_count();
// after n kernel launches: their launch error, else count them globally and in the statistics `launches` of the
// call in flight
inline int launched(int *launches, int n = 1) {
    CUDA_TRY(cudaGetLastError());
    count_launch(n);
    *launches += n;
    return SKB_OK;
}

// Large host -> device copy from PAGEABLE caller memory (per-timestep operator uploads, hundreds of MB): the bytes are
// moved into pinned staging buffers by several host threads while the previous chunk is on the PCIe bus, instead of
// the driver's single-threaded staging path.  Synchronous for the host buffer (it may be reused on return); the device
// side is ordered on `st`.
int upload_pageable(void *d_dst, const void *h_src, size_t bytes, cudaStream_t st);

// Takes device `dev` into use, once per device and process: rejects anything but compute capability 9.0 and loads the
// kernels that need launch attributes, with those attributes set.  Makes `dev` current.
int prepare_device(int dev);
// the launch attributes of the kernels of fiber_ops.cuh and fiber_build.cuh (skb_fiber.cu); called by prepare_device
int prepare_fiber_kernels();
// ... and of the symmetric and cross kernels (skb_sym.cu)
int prepare_sym_kernels();
DeviceInfo query_device(int dev); // (of a prepared device)
LaunchPlan plan_launch(const DeviceInfo &di, int kind, long long n_trg, int n_src_tiles, int force_T, int force_S);
int launch_pair_sum(const DeviceInfo &di, int kind, const double *d_r_src, const double *d_f_packed, long long n_src,
                    long long n_src_pad, const double *d_r_trg, long long n_trg, double *d_partial,
                    const LaunchPlan &plan, cudaStream_t st, const int *d_src_fid = nullptr,
                    const int *d_trg_fid = nullptr);
// width: outputs per target (3, or 10 for the gradient kinds)
int launch_reduce(const double *d_partial, double *d_u, long long n_trg, int n_splits, double scale, int accumulate,
                  cudaStream_t st, int width = 3);

// kRaw: strengths as the caller ships them (3 or 9 per source); kNormalDensity: density, stresslet formed on the device;
// kPacked: already in the kernels' packed, padded layout ([n_pad*3] weighted Stokeslet strengths / [n_pad*6] sym6
// stresslet combinations), e.g. the landing zone peers pushed into -- no pack kernel runs
enum StrengthMode { kRaw = 0, kNormalDensity = 1, kPacked = 2 };

struct EvalOpts {
    double *d_u_sym = nullptr; // symmetric path: write the leading (self-interaction) rows here instead of d_u_out
    int sym_accumulate = -1;   // -1: same as `accumulate`
    double *d_u_rem = nullptr; // symmetric path: write the rows beyond the self-interaction block here instead of
                               // d_u_out + 3 n_src (group mode: the leading rows are partial sums that live elsewhere)
};

constexpr int kMaxGroup = 16; // members of a multi-GPU group (Group, group_kernels.cuh, skb_mflow)
constexpr int kMaxKrylov = 1024; // the largest num_blocks of a solve (SKB_GMRES_MAX_BLOCKS)
constexpr int kDotsSlot = kMaxKrylov + 2; // dots one reduction carries: k + 1 basis columns and a norm

// A member's owned rows of the body part of the solution vector (distributed.system_rows): body node rows [b0, b1)
// (3 each) and the six rows [U; w] of every body whose first node lies in [b0, b1), as runs of consecutive entries in
// ascending order, adjacent runs merged.  At most three: the tail of a body cut at b0 (its six rows belong to the member
// that holds its first node), the bodies that follow up to the one cut at b1, and that body's six rows.
constexpr int kMaxRowPieces = 3;
struct RowPiece {
    long long local, body, len; // local-vector offset (within the body part), body-part offset, length
};
// the pieces of body rows [b0, b1) over bodies of n_nodes[0..n_bodies) nodes; false if they do not fit kMaxRowPieces
bool body_row_pieces(const int *n_nodes, int n_bodies, long long b0, long long b1, std::vector<RowPiece> &out);

// forces_torques [6 x n_bodies] (body_container.cpp:134) -> forces and torques, 3 x n_bodies each
void split_forces_torques(const double *ft, int n_bodies, std::vector<double> &f, std::vector<double> &t);

// ---- per-fiber dense operators of a flow (SURVEY.md §8f N2; skb_fiber.cu) ----
// The fibers whose operators are resident (the fiber rows of the flow's target list) and what the build reads
struct OwnFibers {
    int f0 = 0, f1 = 0;             // fibers [f0, f1)
    const int *n = nullptr;         // node count of every fiber of the flow
    const long long *off = nullptr; // first node of every fiber of the flow (n_fibers + 1 entries)
    const double *r_fib = nullptr;  // device: positions of all fiber nodes
    const double *length = nullptr; // device: length of every fiber
    cudaStream_t stream = nullptr;  // uploads, the build and the read-back are ordered on it
    int count() const { return f1 - f0; }
    long long nodes() const { return f1 > f0 ? off[f1] - off[f0] : 0; }
};

struct FiberItem; // fiber_build.cuh
// a fiber of the fiber step (step_kernels.cuh), as FiberOps::step_items fills it and the step places it
struct StepItem {
    long long node;  // first node of the fiber among the launch's nodes (positions 3 per node, solution 4 per node)
    long long d1;    // element offset of its class's D_1_0 (n x n, column-major) in the class table
    long long rng;   // offset of its class's D_1_0 column ranges (int2 per column) in the class ranges
    double site[3];  // the lab-frame nucleation site a bound fiber is repinned to
    int n;           // nodes
    int bound;       // 1: repin to site
};

// one body of the solution vector, in the order of skb_flow_set_bodies (body_ops.cuh, listener_kernels.cuh)
struct BodyItem {
    long long node_off; // first node among all body nodes
    long long sol_off;  // first entry in x_bodies: [densities (3n) | U (3) | w (3)]
    int n_nodes, pad;
};

// A_, force_operator_, xs_ and A_^-1 of one set of own fibers, resident for the timestep, and the GEMVs over them.
// The caller has checked its pointers for NULL and made the flow's device current.
class FiberOps {
  public:
    // the class matrices of n_nodes, uploaded at once on st after the device has drained (the GEMVs, the build and the
    // RHS read them on any stream); set_class drops the operators
    int set_class(int n_nodes, const double *D_1_0, const double *P_downsample_bc, cudaStream_t st);
    int set_class_derivatives(int n_nodes, const double *D_2_0, const double *D_3_0, const double *D_4_0,
                              cudaStream_t st);
    int upload(const OwnFibers &own, const double *A, const double *force_operator, const double *xs,
               const double *length_prev, const int *plus_bc_velocity);
    int upload_inverse(const double *A_inv, cudaStream_t st);
    // the device build, checked and planned on the host first; `frame` runs stage (the table uploads), then launch
    // (assembly and inverse kernels, adding to *launches) and returns once own.stream has drained.  No own fibers:
    // the empty set, without a frame.  with_inverse false: A_, force_operator_ and xs_ only, and the preconditioner
    // refuses (ready(who, true)) until a build with the inverse
    using Step = std::function<int()>;
    int build(const OwnFibers &own, const ::skb_fiber_params *params, double dt, double eta, int *launches,
              const std::function<int(const Step &stage, const Step &launch)> &frame, bool with_inverse = true);
    // the fiber block of the RHS into d_rhs (4 per own node) from d_v / d_f (3 per own node, either may be NULL),
    // checked on the host first; `frame` runs stage (the table uploads on own.stream), then launch.  Needs the class
    // matrices and derivatives, not the operators: its per-fiber tables are its own, and the resident operators, their
    // inverse and the GEMV launches stay as they are.  v_growth / force_scale per own fiber, may be NULL
    int rhs(const OwnFibers &own, const ::skb_fiber_params *params, const double *v_growth, const double *force_scale,
            const double *d_v, const double *d_f, double dt, double eta, double *d_rhs, int *launches,
            const std::function<int(const Step &stage, const Step &launch)> &frame);
    // on st, each adding its launches to *launches: fw = force_operator_ x; res = fc.matvec(x, v, vb); y = A_^-1 x
    int force(const double *d_x, double *d_fw, cudaStream_t st, int *launches) const;
    int matvec(const double *d_x, const double *d_v, const double *d_vb, double *d_res, cudaStream_t st,
               int *launches) const;
    int precondition(const double *d_x, double *d_y, cudaStream_t st, int *launches) const;
    int read(double *A, double *force_operator, double *xs, double *A_inv, cudaStream_t st) const; // any may be NULL
    // the per-fiber tables and the event of rhs() for n_fibers own fibers, at their final size (a group member's RHS
    // must not allocate once its peers may wait on a flag)
    int size_rhs(int n_fibers);
    // every buffer build() fills for the fibers `own` at its final size, and the assembly kernel loaded (a group step
    // builds while its peers may wait on a flag); nothing is sized while a class the build needs is missing, and then
    // build_sized_for(own) stays false
    int size_build(const OwnFibers &own);
    bool build_sized_for(const OwnFibers &own) const { return build_key_ == build_key(own); }
    int ready(const char *who, bool with_inverse = false) const; // an error naming `who` unless they are resident
    // a fiber of n nodes can be built: n within the build's range, skb_flow_set_fiber_class(n) and
    // skb_flow_set_fiber_class_derivatives(n) called
    bool buildable(int n) const;
    static int build_min_nodes();
    static int build_max_nodes();
    bool empty() const { return n_items_A == 0; }
    int n_fibers() const { return f1 - f0; }
    // drops the resident operators: no GEMV runs on them again (a flow left with no fibers has the empty set)
    void invalidate() {
        ready_ = false;
        n_items_A = n_items_F = 0;
    }
    // what the fiber-body links read (BodyOps): the element offset of D_2_0 of fiber f's class (n nodes) in the class
    // table, D_3_0 following -- an error unless skb_flow_set_fiber_class_derivatives(n) was called; offsets move when
    // set_class adds a node count.  The table and the resident tangents xs_ (3 per own node) on the device
    int derivative_offset(int f, int n, long long *off) const;
    const double *class_table() const { return (const double *)class_mats.ptr; }
    const int2 *class_range_table() const { return (const int2 *)class_ranges.ptr; }
    // the fiber step's item of every own fiber (step_kernels.cuh: its D_1_0 and their column ranges; node offsets from
    // the first own node, free); an error unless each node count has skb_flow_set_fiber_class and at most
    // kStepMaxNodes nodes
    int step_items(const OwnFibers &own, std::vector<StepItem> &items) const;
    // the refusals of build() and rhs() for these arguments, without a launch or a change of state
    int check_step(const OwnFibers &own, const ::skb_fiber_params *params, const double *v_growth,
                   const double *force_scale) const;
    const double *tangents() const { return (const double *)op_xs.ptr; }

  private:
    struct Plan;
    int plan(const OwnFibers &own, const double *length_prev, const ::skb_fiber_params *build, Plan &pl);
    int upload_plan(const OwnFibers &own, const Plan &pl);
    void commit(const OwnFibers &own, const Plan &pl);

    struct FiberClass {
        std::vector<double> D, P; // D_1_0 (n x n), P_downsample_bc ((4n-14) x 4n), column-major
        std::vector<double> D234; // D_2_0 | D_3_0 | D_4_0 (n x n each): set_class_derivatives
    };
    int upload_classes(cudaStream_t st);
    int check_class(int f, int n, bool derivatives) const; // fiber f has n nodes: its class is set
    int item(const OwnFibers &own, int f, bool derivatives, FiberItem &it) const; // own fiber f, check_class first
    std::map<int, FiberClass> classes;
    // the device copy of `classes` (upload_classes): per n with set_class a block [D_1_0 | P_downsample_bc | D_2_0 |
    // D_3_0 | D_4_0], the last three zero until set_class_derivatives, so that a block's offset depends only on which
    // n have set_class; and the non-zero ranges of P's rows and D_1_0's columns.  class_off[n]: offsets of both
    std::map<int, std::pair<long long, long long>> class_off;
    DevBuf class_mats, class_ranges;
    bool ready_ = false;
    int f0 = 0, f1 = 0;    // the fibers of the resident operators
    long long n_nodes = 0; // ... and their nodes
    int n_items_A = 0, n_items_F = 0;
    size_t gemv_smem = 0;
    DevBuf op_A, op_F, op_xs, op_Ainv, op_len, op_plus, op_classD, op_classP, op_classR, items_A, items_F, bld_params,
        bld_items, bld_tiles, bld_inv;
    long long op_A_elems = 0;                        // elements of the concatenated A_ (and of A_^-1)
    long long op_F_elems = 0;                        // ... of force_operator_
    unsigned long long ops_gen = 0, precond_gen = 0; // the inverse belongs to one set of operators
    // the RHS's per-fiber tables of the last call, and the event after its kernel (the next call's uploads wait for it)
    DevBuf rhs_items, rhs_params, rhs_growth;
    Event rhs_done;
    bool rhs_pending = false;
    // the fibers and nodes size_build sized for
    static std::array<long long, 4> build_key(const OwnFibers &own) {
        return {own.f0, own.f1, own.count() > 0 ? own.off[own.f0] : 0, own.nodes()};
    }
    std::array<long long, 4> build_key_ = {-1, -1, -1, -1};
};

struct FiberGemvItem; // fiber_ops.cuh
// y = M x per item with fiber_gemv_kernel<0> (launched from skb_fiber.cu, which sets its shared-memory limit), adding
// one launch to *launches; smem = fiber_gemv_kernel's dynamic shared memory for the widest item
int launch_gemv(const FiberGemvItem *d_items, int n_items, const double *mats, const double *x, double *y, size_t smem,
                cudaStream_t st, int *launches);

// ---- the bodies' per-timestep operators and the fiber-body links of a single-device flow (skb_body.cu) ----
// The body block of System::apply_matvec / ::apply_preconditioner (BodyContainer::matvec / ::apply_preconditioner,
// body_container.cpp:487-521) and BodyContainer::calculate_link_conditions (:171-267), on the device.  Bodies are in
// the order of skb_flow_set_bodies, which is the order of the solution vector.  The caller has checked its pointers
// for NULL and made the flow's device current; every step runs on the stream it passes.
//
// A group member (skb_mflow) owns the body node rows [lo, hi) of the solution vector -- 3 rows each -- and the six rows
// [U; w] of every body whose FIRST node lies in [lo, hi); it keeps the inverses of the bodies it owns rows of, and
// matvec / precondition write those rows only (of an output in the complete body layout).
class BodyOps {
  public:
    // per body: n_nodes (summing to n_body_nodes), node_weights_, ex_ / ey_ / ez_ (3 per node), A_^-1 (column-major
    // (3n+6)^2, concatenated; may be NULL); r_body / centers: the flow's geometry (host).  hi >= 0: a member's body
    // node rows [lo, hi).  Checked first: a refusal leaves the earlier operators
    int set_operators(const int *n_nodes, int n_bodies, long long n_body_nodes, const double *r_body,
                      const double *centers, const double *node_weights, const double *ex, const double *ey,
                      const double *ez, const double *A_inv, cudaStream_t st, long long lo = 0, long long hi = -1);
    // per fiber of `own` (all fibers of the flow, or a member's own fibers): body index (-1 free; body == NULL: none
    // bound), lab-frame nucleation site, bending_rigidity_.  Checked first: a refusal leaves the earlier links;
    // check_only: the checks and nothing else
    int set_links(const OwnFibers &own, const FiberOps &ops, int n_bodies, const double *centers, const int *body,
                  const double *site, const double *rigidity, cudaStream_t st, bool check_only = false);
    // every buffer set_links fills, at its size for n_fibers fibers (all of them bound) and n_bodies bodies: a later
    // set_links of as many fibers allocates nothing (a group step sets the links while its peers may wait on a flag)
    int size_links(int n_fibers, int n_bodies);
    // The body frame of rigid bodies (skb_flow_set_body_frames): per body n_nodes (summing to n_body_nodes), the
    // reference nodes, normals and weights (3, 3, 1 per node), ex_ / ey_ / ez_ and A_^-1 (may be NULL) at identity
    // orientation.  Kept resident next to the placed operators, the inverses of the bodies a member owns rows of only;
    // sizes every buffer set_operators and place use and loads the placement kernel, and drops the placed operators.
    // Checked first: a refusal leaves the earlier frames and operators
    int set_frames(const int *n_nodes, int n_bodies, long long n_body_nodes, const double *pos_ref,
                   const double *normal_ref, const double *node_weights, const double *ex0, const double *ey0,
                   const double *ez0, const double *A_inv0, cudaStream_t st, long long lo = 0, long long hi = -1);
    bool has_frames() const { return frames_set_; }
    int frame_bodies() const { return (int)frame_n_.size(); }
    long long frame_nodes() const { return (long long)frame_w_.size(); }
    const int *frame_node_counts() const { return frame_n_.data(); }
    bool frame_window(long long lo, long long hi) const { return frame_lo_ == lo && frame_hi_ == hi; }
    // the nodes and normals at rotations R (9 per body, row-major) and centres: x_i = c + R r_i, n_i = R n_i,ref
    void placed_geometry(const double *R, const double *centers, std::vector<double> &pos,
                         std::vector<double> &normals) const;
    // the operators of the frames at rotations R, with r_body / centers the flow's geometry (placed_geometry): the
    // state set_operators would leave with the placed operators; allocates nothing.  The caller has checked that
    // the frames match the flow's bodies
    int place(const double *R, const double *r_body, const double *centers, cudaStream_t st);
    // the resident ex_ / ey_ / ez_ (3 per node) and the kept inverses (concatenated, column-major); NULL skips one
    int read(double *ex, double *ey, double *ez, double *A_inv, cudaStream_t st) const;
    long long kept_inverse_elements() const { return inv_own_; }

    void drop_operators() { ops_set_ = false; }
    void drop_links() { links_set_ = false; }
    bool has_operators() const { return ops_set_; }
    bool has_inverse() const { return ops_set_ && inv_set_; }
    bool has_links() const { return links_set_; }
    long long solution_size() const { return sol_size_; }

    // one matvec: the link conditions (*d_link: 7 per fiber, NULL when no fiber is bound), the bodies' link forces /
    // torques and their densities gathered from x_bodies (forces(), torques(), densities()).  length: length_ per fiber.
    // Over a member's own fibers the forces and torques are its partial sums
    int links(const FiberOps &ops, const double *d_length, const double *d_x_fib, const double *d_x_bodies,
              const double **d_link, cudaStream_t st, int *launches);
    const BodyItem *items() const { return (const BodyItem *)items_.ptr; } // per body, on the device
    const double *densities() const { return (const double *)dens_.ptr; }
    const double *forces() const { return (const double *)force_.ptr; }
    const double *torques() const { return (const double *)torque_.ptr; }
    // res_bodies = bc.matvec(v_bodies, x_bodies); y = A_^-1 x per body.  A member's precondition evaluates every
    // 32-row block of a body's GEMV that reaches one of its rows: the other rows of such a block are written to d_y as
    // well and are scratch -- only the member's own rows of d_y are results
    int matvec(const double *d_x_bodies, const double *d_v_bodies, double *d_res, cudaStream_t st,
               int *launches) const;
    int precondition(const double *d_x, double *d_y, cudaStream_t st, int *launches) const;
    // the shell and body rows of the RHS in one launch: d_rhs_shell = -d_v_shell (n_shell_rows rows) and, with
    // `bodies`, per body [-v of its nodes ; 0 x 6] into d_rhs_bodies (x_bodies layout, the rows matvec writes) from
    // d_v_bodies (the body rows matvec reads)
    int rhs_rows(bool bodies, const double *d_v_bodies, double *d_rhs_bodies, const double *d_v_shell,
                 long long n_shell_rows, double *d_rhs_shell, cudaStream_t st, int *launches) const;

  private:
    struct Plan; // the layout of one set of node counts and row window (skb_body.cu)
    int plan(const char *who, const int *n_nodes, int n_bodies, long long n_body_nodes, const double *node_weights,
             bool with_inverse, long long lo, long long hi, Plan &pl) const;
    int upload_layout(const Plan &pl, const double *r_body, const double *centers, const double *node_weights,
                      cudaStream_t st);
    void commit(const Plan &pl, bool with_inverse);

    bool ops_set_ = false, inv_set_ = false, links_set_ = false, any_bound_ = false;
    int n_bodies_ = 0, n_fibers_ = 0, n_gemv_ = 0;
    long long sol_size_ = 0, inv_own_ = 0;
    // the frames: host copies of what place needs, the placement table of the kept inverses
    bool frames_set_ = false, frame_inv_ = false;
    std::vector<int> frame_n_;
    std::vector<double> frame_r_, frame_nrm_, frame_w_;
    long long frame_lo_ = 0, frame_hi_ = -1;
    int n_place_ = 0, place_ctas_ = 0;
    DevBuf ex0_, ey0_, ez0_, a_inv0_, place_items_, rot_;
    bool windowed_ = false; // a member's rows: bodies [win_b0_, win_b1_) have nodes in [win_lo_, win_hi_)
    int win_b0_ = 0, win_b1_ = 0;
    long long win_lo_ = 0, win_hi_ = 0;
    size_t gemv_smem_ = 0;
    DevBuf items_, r_, centers_, weights_, ex_, ey_, ez_, a_inv_, gemv_items_; // set_operators
    DevBuf link_fibers_, csr_begin_, csr_fib_, link_, contrib_;                 // set_links
    DevBuf dens_, force_, torque_;                                              // per matvec
};
// loads the kernel of BodyOps::rhs_rows (a group member's first launch must not load it lazily)
int load_rhs_rows_kernel();
// loads the kernel of skb_dense_apply_device (skb_dense.cu), for the same reason: a kernel loaded lazily while a peer on
// the same device spins on a flag waits for that peer, which waits for this member
int load_dense_kernels();

// ---- one member of a multi-GPU group of flows (DESIGN.md §4; skb_group.cu, group_kernels.cuh) ----
// A group is one flow per GPU exchanging strengths and partial velocities through peer memory.  Every member owns a
// WINDOW of device memory that all members can address, laid out by init (each piece 256-byte aligned):
//
//   flags        [5][kMaxGroup] + 8  epoch counters, one slot per (phase, writer); then the error word (0, or
//                                    1 + the rank a flag wait gave up on)                        -- written by peers
//   f_sl         [2][n_pad_fib*3]    packed (trapezoid-weighted) Stokeslet strengths of ALL fiber nodes   -- by peers
//   f_shell      [2][n_pad_shell*6]  packed sym6 stresslet strengths of ALL periphery nodes                -- by peers
//   x_shell      [2][n_shell*3]      periphery density of ALL nodes (input of the dense operator; the matvec's push
//                                    and the rank-per-GPU preconditioner's row store write it)    -- by peers
//   ft_part      [2][kMaxGroup][n_bodies*6]  per member its partial link forces / torques of ALL bodies
//                                    ([F | L]; the whole-vector operator, skb_mflow_apply_system_matvec) -- by peers
//   x_body       [2][n_body*3 + n_bodies*6]  the body part of the solution vector, complete (every member stores
//                                    its own rows; skb_flow_group_apply_system_*)                   -- by peers
//   dots         [2][kMaxGroup][kDotsSlot]  per member its partial dot products of a solve step (reduce_dots)
//                                    -- by peers
//   r_step       [2][n_fib*3 + 2*n_fibers]  the new positions of ALL fiber nodes, the errors of ALL fibers and, with a
//                                    periphery shape, their minus_clamped flags after a group step
//                                    (skb_flow_group_step_device; group_fiber_step_kernel)             -- by peers
//   u_part       [n_fib*3]           this member's partial velocities of ALL fiber rows                  -- by itself
//   u_part_shell [n_shell*3]         its partial velocities of ALL periphery rows (cross kernel)        -- by itself
//
// [2]: double buffering by epoch parity -- a peer may already push the next call's strengths or rows while this member
// still reads the current ones (DESIGN.md §4 argues why the other half is never still being read).  A
// default-constructed Group is no member (size 1).  Knows nothing of the flow: the caller has made the flow's device
// current, and every step runs on the stream it passes, adding its launches to *launches.
class Group {
  public:
    // allocates and zeroes the window of member `rank` of `size` for that many fiber / periphery / body nodes, bodies
    // and fibers; n_pad_*: the padded source counts of the flow's evaluators (the window replaces their packed
    // strengths).  Size 1: no member
    int init(int rank, int size, long long n_fib, long long n_pad_fib, long long n_shell, long long n_pad_shell,
             long long n_body, int n_bodies, int n_fibers);
    int export_handle(void *handle) const;                     // the window's CUDA-IPC handle
    int import_handle(int peer_rank, const void *handle);      // maps another process's member's window
    int connect(int peer_rank, const Group &peer, int dev, int peer_dev); // a member in this process, on peer_dev
    int missing_peer(int *missing) const; // -1, or the rank a flag wait gave up on (no window: -1)

    bool member() const { return size_ > 1; }
    bool has_window() const { return window_.get() != nullptr; }
    int rank() const { return rank_; }
    int size() const { return size_; }
    // an error unless laid out for these
    int check_layout(long long n_fib, long long n_shell, long long n_body, int n_bodies, int n_fibers) const;
    // solo (warm-up, profiling): no flags, push and pull over this member's own window only, no connectedness check
    void set_solo(bool solo) { solo_ = solo; }
    void restart() { epoch_ = 0; } // the next matvec is the group's first

    // ---- one matvec: begin, push, barrier(0), pair kernels, barrier(1), pull ----
    int connected() const; // an error unless every peer's window is mapped (solo: always)
    int begin(); // refuses a member whose peers are not all connected; advances the epoch (its parity picks the half)
    // pack the own strengths once and store them into every window: fiber forces d_fw [n_f*3] of nodes [fa, fa + n_f)
    // (weighted by d_weight of ALL fiber nodes, NULL: 1), periphery densities d_density [n_s*3] of rows [sa, sa + n_s)
    // (sym6 with two_eta and d_normal of ALL periphery nodes, and raw into x_shell)
    int push(const double *d_fw, const double *d_weight, long long fa, long long n_f, const double *d_density,
             const double *d_normal, long long sa, long long n_s, double two_eta, int num_sms, cudaStream_t st,
             int *launches) const;
    int barrier(int phase, bool signal, bool wait, cudaStream_t st, int *launches) const;
    // the bodies' link forces of the whole-vector operator: push_forces stores this member's partials d_f / d_t
    // [n_bodies*3 each] into its slot of every window (before barrier 0); reduce_forces (after it) writes the sum of
    // every member's slot, in rank order, to d_f / d_t
    int push_forces(const double *d_f, const double *d_t, cudaStream_t st, int *launches) const;
    int reduce_forces(double *d_f, double *d_t, cudaStream_t st, int *launches) const;
    // d_v rows [0, n_rows) += the sum of every member's partial rows [row0, row0 + n_rows), in rank order
    enum Partials { kFiberRows, kShellRows };
    int pull(Partials which, long long row0, long long n_rows, double *d_v, cudaStream_t st, int *launches) const;

    // ---- a rank-per-GPU member's own rows of the solution vector (skb_flow_group_* whole-vector calls) ----
    // the member's resolved target ranges: fiber nodes [fa, fb), periphery rows [sa, sb), body nodes [ba, bb)
    using Ranges = std::array<long long, 6>;
    // the pieces of its body rows [ba, bb) (body_row_pieces), kept until init, and the ranges the caller sized its
    // buffers for; rows_for: they were set for exactly these ranges (any other split of the rows wants the set-up again)
    void set_body_rows(const std::vector<RowPiece> &pieces, const Ranges &ranges);
    bool rows_for(const Ranges &ranges) const { return rows_set_ && rows_ranges_ == ranges; }
    long long body_rows() const { return rows_.total; } // own body rows of the local vector
    // d_body [body_rows()] into x_body of every window at the pieces' places, and (d_shell != NULL) the own periphery
    // rows d_shell [n_s*3] of rows [sa, sa + n_s) into x_shell, in one kernel (before the rows phase's barrier)
    int store_rows(const double *d_body, const double *d_shell, long long sa, long long n_s, int num_sms,
                   cudaStream_t st, int *launches) const;
    int rows_barrier(bool signal, bool wait, cudaStream_t st, int *launches) const; // barrier of the rows phase
    // d_local [body_rows()] = the own rows of d_full (the whole body layout)
    int compact_rows(const double *d_full, double *d_local, cudaStream_t st, int *launches) const;
    // the all-reduce of a solve's dot products, one epoch of its own (begin, the dots phase's full barrier): d_v[0, m) =
    // the sum over every member's d_v in rank order, bitwise the same on every member.  Not a member: nothing to do
    int reduce_dots(double *d_v, int m, cudaStream_t st, int *launches);

    // ---- the all-gather of a group step's new fiber positions and errors (skb_flow_group_step_device) ----
    // r_step of every window the step's store reaches, in the current epoch's half (solo: the own one only); returns
    // their count.  The store is group_fiber_step_kernel itself; then the rows phase's barrier, in the step's epoch
    int step_windows(double **r_step) const;

    // this member's window, in the half of the matvec in flight
    double *f_sl() const { return own(lay_.f_sl[epoch_ & 1]); }
    double *f_shell() const { return own(lay_.f_shell[epoch_ & 1]); }
    double *x_shell() const { return own(lay_.x_shell[epoch_ & 1]); }
    double *x_body() const { return own(lay_.x_body[epoch_ & 1]); }
    double *r_step() const { return own(lay_.r_step[epoch_ & 1]); }
    double *u_part() const { return own(lay_.u_part); }
    double *u_part_shell() const { return own(lay_.u_part_shell); }

  private:
    struct Layout { // byte offsets of the window's pieces
        size_t flags = 0, f_sl[2] = {0, 0}, f_shell[2] = {0, 0}, x_shell[2] = {0, 0}, ft_part[2] = {0, 0},
               x_body[2] = {0, 0}, dots[2] = {0, 0}, r_step[2] = {0, 0}, u_part = 0, u_part_shell = 0;
        size_t bytes = 0;
    };
    struct Rows { // the piece table of set_body_rows, as the kernels take it (RowPiecesDev, group_kernels.cuh)
        long long local[kMaxRowPieces] = {}, body[kMaxRowPieces] = {}, len[kMaxRowPieces] = {};
        int n = 0;
        long long total = 0;
    };
    double *own(size_t off) const { return reinterpret_cast<double *>((char *)window_.get() + off); }
    int windows(char **w) const; // the windows push and pull reach (solo: the own one only); returns their count

    int rank_ = 0, size_ = 1;
    DevPtr window_;              // this member's window (cudaMalloc: exportable through CUDA IPC)
    Layout lay_;
    void *peer_[kMaxGroup] = {}; // every member's window as mapped here (peer_[rank_] == window_)
    IpcPtr ipc_[kMaxGroup];      // the windows of other processes' members that this one has mapped
    long long n_fib_ = 0, n_shell_ = 0, n_body_ = 0; // geometry the window was laid out for
    int n_bodies_ = 0, n_fibers_ = 0;
    unsigned long long epoch_ = 0;
    bool solo_ = false;
    Rows rows_;
    bool rows_set_ = false;
    Ranges rows_ranges_ = {};
};

// ---- right-preconditioned restarted GMRES on the device (skb_solve.cu, krylov_kernels.cuh) ----
// The workspace of one solution size -- the basis V of (num_blocks + 1) columns, the per-CTA dot partials, the
// Hessenberg scalars and the pinned words the host reads once per Arnoldi step -- and the iteration over two operators
// given as calls on the solve's stream.  Givens rotations, the triangular solve and every stopping decision run on the
// host from the words the device reduced in a fixed order.
class Krylov {
  public:
    // sizes everything for n rows (0 allowed: a group member that owns none still takes part in every reduction) and
    // up to num_blocks basis vectors per cycle on the current device (num_sms: its SMs, which fix the reduction grid),
    // and loads the kernels; key: what else the size belongs to (a member's target ranges).  A set-up call: allocates
    int setup(long long n, int num_blocks, int num_sms, const std::array<long long, 6> &key);
    bool sized_for(long long n, const std::array<long long, 6> &key) const { return set_ && n_ == n && key_ == key; }
    int blocks() const { return m_cap_; }
    // the host forms' copies of b and x (n doubles each), sized by setup
    double *stage_b() const { return (double *)b_.ptr; }
    double *stage_x() const { return (double *)x_.ptr; }
    // out = A in / P^-1 in, enqueued on the solve's stream
    using Apply = std::function<int(const double *d_in, double *d_out)>;
    // d_v[0, m) (device, on the solve's stream) = the sum of every member's d_v: the all-reduce of a group member
    // (Group::reduce_dots); empty for a single flow
    using Reduce = std::function<int(double *d_v, int m)>;
    // x = the GMRES solution of A x = b (x0 = 0, right preconditioning, ICGS); d_x is written, d_b only read.  info
    // (skb_solve_info) and history (iterations + 1 implicit relative residuals, may be NULL) as skb_flow_solve_system
    // documents them.  Each launch adds to *launches.  The host waits for one event per Arnoldi step and per cycle end
    int solve(const Apply &A, const Apply &P_inv, const Reduce &reduce, const double *d_b, double *d_x, double tol,
              int num_blocks, int max_iters, cudaStream_t st, ::skb_solve_info *info, double *history, int *launches);

  private:
    int pass(int which, int k, double *d_w, const double *d_coef, double *d_out, const Reduce &reduce,
             cudaStream_t st, int *launches);
    // V col 0 = b - ax, its norm^2 -> nrm[1]
    int residual(const double *d_b, const double *d_ax, const Reduce &reduce, cudaStream_t st, int *launches);
    int wait(cudaStream_t st); // the device words -> host_, then one event wait

    bool set_ = false;
    long long n_ = 0, ld_ = 0, rows_per_ = 0;
    std::array<long long, 6> key_ = {};
    int m_cap_ = 0, ctas_ = 0, ldp_ = 0;
    DevBuf V_, z_, u_, part_, small_, b_, x_;
    PinnedHost host_;
    Event done_;
    std::vector<double> H_, cs_, sn_, g_, y_; // the Hessenberg matrix ((m + 1) x m, column-major) and its rotations
};

// ---- the symmetric and cross pair kernels' host side (skb_sym.cu, sym_kernels.cuh, cross_kernels.cuh) ----
// One launch of either kernel on the device: its work items in launch order, row_begin (the items of every block row),
// one forward-partial slab per item (F) and the reverse partials (P)
struct ItemPlan {
    DevBuf items, row_begin, F, P;
    int n_items = 0, n_blocks = 0;
};
// The symmetric path of one set of Stokeslet sources: the plan of key (nb, part, parts) and what only it keeps
struct SymState {
    int self_state = -1; // -1 unknown, 0 targets do not start with these sources, 1 they do
    ItemPlan plan;
    std::array<int, 3> key = {0, 0, 0};
    DevBuf row_ids, flag; // block row I of every row of P; the answer of the self check
    int n_owned = 0;      // rows of P
    long long pairs = 0;  // ordered (target, source) pairs one launch covers (both directions)
};
// The cross kernel's plan of key (node0, n_rows, n_sh, n_sh_pad, num_sms): one (fiber rows, periphery) shape
struct CrossState {
    ItemPlan plan;
    std::array<long long, 5> key = {-1, -1, -1, -1, -1};
};

// One set of sources of an Evaluator: Stokeslet (kind 0) or stresslet (kind 1)
struct SourceSet {
    long long n = -1; // -1 = never set
    long long n_pad = 0;
    bool has_normals = false;
    DevBuf r;       // padded positions
    bool has_weights = false;
    DevBuf normals; // optional (double layer formed on device)
    DevBuf weights; // optional per-source quadrature weight folded into the Stokeslet strengths
    DevBuf f_raw;   // strengths as shipped by the caller (3 or 9 per source; all-gather landing zone)
    DevBuf f_packed;
    const double *f_cur = nullptr; // packed strengths of the evaluation in flight (f_packed, or the caller's kPacked buffer)
    // opt-in fused self-exclusion (SURVEY.md 8f N3): Stokeslet sources and the leading targets carry an id (the fiber
    // index); pairs with equal ids contribute 0.  excl_ids: [n_pad] source ids; excl_trg: [n_trg] target ids (-1 beyond
    // the leading n targets), built on demand for the plain kernel
    bool excl = false;
    DevBuf excl_ids, excl_trg;
    long long excl_trg_n = -1;
    SymState sym; // symmetric (Newton's third law) path of the Stokeslet self-interaction
};

// The pair sums of one device (skb_runtime.cu; the symmetric path: skb_sym.cu): its targets, both sets of sources and
// the buffers and streams of the plain and symmetric kernels.  A flow holds six, a context (skb_ctx.cu) one per device.
// The setters enqueue their copies on the stream the caller passes and do not wait for them; the caller synchronises
// before a host buffer it passed goes out of scope.
struct Evaluator {
    DeviceInfo info;
    long long trg_begin = 0, n_trg = 0; // this device's block of the caller's target list
    DevBuf r_trg, partial, scratch;
    SourceSet src[2];
    Stream aux_stream; // remainder targets run beside the symmetric kernel (created on its first use)
    Event ev_fork, ev_join;
    Event ev_s0, ev_s1; // around the symmetric kernel's launch (its live duration inside a step)
    bool sym_timed = false;
    int sym_part = 0, sym_parts = 1; // block rows of the self-interaction this device evaluates
    // how it evaluates
    int force_T = 0, force_S = 0;
    int sym_mode = -1; // -1 auto, 0 never, 1 whenever the sources are the leading targets
    // kOwn: the targets are this evaluator's alone; a multi-device context's plain block layout (kBlocks) takes neither
    // the symmetric path nor the device's exclusion check, and its symmetric layout (kShared) reduce-scatters the
    // leading rows' partial sums, so the symmetric path may not decline there
    enum Layout { kOwn, kBlocks, kShared } layout = kOwn;
    bool last_was_sym = false; // the last Stokeslet evaluation took the symmetric path

    // on device di.dev, prepared and current: the symmetric path's events; sym_mode from SKB_SYMMETRIC
    int init(const DeviceInfo &di);
    // n targets [3 n] from host or device memory, all of them this evaluator's (trg_begin 0)
    int set_targets(const double *r, long long n, bool on_device, cudaStream_t st);
    // n sources of `kind`; f_raw holds n_parts slots of ceil(n / n_parts) sources (a context's all-gather)
    int set_sources(int kind, const double *r, long long n, bool on_device, cudaStream_t st, long long n_parts = 1);
    int set_normals(const double *normals, long long n, cudaStream_t st); // of the stresslet sources (host)
    int set_exclusion_ids(const int32_t *ids, long long n, cudaStream_t st); // of the Stokeslet sources (host); NULL: off
    // strengths -> the kernels' packed, padded layout in s.f_packed (what eval does first); sets s.f_cur
    int pack(int kind, StrengthMode mode, const double *d_f_raw, double two_eta, cudaStream_t st, int *launches);
    // pack -> pair sums -> split reduction; strengths already resident at d_f_raw.
    // result (=|+=) scale_mul * [1 | -3]/(8 pi) * sum.  ev_k0 / ev_k1, when given, are recorded around the pair sums
    int eval(int kind, StrengthMode mode, const double *d_f_raw, double two_eta, double *d_u_out, int accumulate,
             cudaStream_t st, int *launches, LaunchPlan *plan_out, double scale_mul, const EvalOpts &opts = EvalOpts(),
             cudaEvent_t ev_k0 = nullptr, cudaEvent_t ev_k1 = nullptr);
    // The velocity gradient and pressure of the sources of `kind` (strengths as eval takes them) at the targets,
    // through the gradient kinds of the plain kernel: d_g[10 t + 3 i + j] += scale_mul * [1 | -3]/(8 pi) * sum of
    // d u_i / d x_j, and d_g[10 t + 9] += the same scale times 2 x the pressure numerator (p / eta when scale_mul is
    // 1 / eta).  Always accumulates; nothing to do without targets or sources.
    int gradient(int kind, StrengthMode mode, const double *d_f_raw, double two_eta, double *d_g, cudaStream_t st,
                 int *launches, double scale_mul);
    // the duration and pairs of the last symmetric kernel, once it has run (0 before)
    int last_sym_kernel(double *ms, int64_t *pairs) const;
};
int check_kind(int kind); // SKB_STOKESLET or SKB_STRESSLET
// the refusals of set_sources' arguments
int check_sources(int kind, const double *r, long long n);
// dfma_probe_kernel on st: blocks x threads, iters FMA chains of 8 into d_out (pair_kernels.cuh)
int launch_fp64_probe(double *d_out, int blocks, int threads, int iters, cudaStream_t st);

// the symmetric and cross kernels (skb_sym.cu)
long long sym_block_nodes(); // nodes per block of the symmetric kernel (its I side)
long long sym_mem_budget();  // bytes its reverse partials may occupy on one device
// are the first n_src targets bit-identical to the Stokeslet sources (s.sym.self_state, decided once per positions)?
int ensure_self_state(Evaluator &e, SourceSet &s, cudaStream_t st);
// Decide whether the symmetric path serves e's Stokeslet sources (*use) and make sure its plan and buffers exist
int sym_prepare(Evaluator &e, cudaStream_t st, int *use);
// u[0 : 3 n_src] (=|+=) scale_mul / (8 pi) * sum over the square block, using the plan above.  Strengths are packed
int sym_eval(Evaluator &ev, double *d_u_out, int accumulate, cudaStream_t st, double scale_mul, int *launches);
LaunchPlan sym_launch_plan(const SourceSet &s); // the last symmetric launch, as the stats report it
// fiber <-> periphery in one geometry pass (cross_kernels.cuh), on the plan of cs (made again for a new shape):
// u_fib[n_rows x 3] (=|+=) scale_dl * (stresslet sums of ALL periphery nodes at fiber nodes [node0, node0 + n_rows));
// u_shell[n_sh x 3] (=|+=) scale_sl * (Stokeslet sums of those fiber nodes at every periphery node).
// r_fib / h: positions and packed Stokeslet strengths of all fiber nodes (padded); r_sh / s6: periphery, padded.
int cross_eval(CrossState &cs, const DeviceInfo &di, const double *d_r_fib, const double *d_h, long long node0,
               long long n_rows, const double *d_r_sh, const double *d_s6, long long n_sh, long long n_sh_pad,
               double scale_dl, double scale_sl, double *d_u_fib, int acc_fib, double *d_u_shell, int acc_shell,
               cudaStream_t st, int *launches);

// NCCL is bound at run time (dlopen "libnccl.so.2"): a single-GPU user never needs it, and a host that
// already loaded NCCL (PyTorch) shares that copy instead of getting a second one.
int nccl_group_create(size_t n, const std::function<int(int)> &device_of, void **out);
int nccl_group_allgather_inplace(void *group, void *const *bufs, size_t count_per_rank_doubles,
                                 const cudaStream_t *streams);
// recv[g] (count doubles) = sum over ranks of send[r][g*count : (g+1)*count]
int nccl_group_reduce_scatter(void *group, void *const *send, void *const *recv, size_t count_per_rank_doubles,
                              const cudaStream_t *streams);
void nccl_group_destroy(void *group);

} // namespace skb

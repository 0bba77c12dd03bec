// skb_system.cu -- the whole-system calls of a flow (include/skelly_b200_flow.h): the fibers' per-fiber operators (class
// tables, upload or device build, RHS and GEMVs), the bodies' operators, frames, placement and the fiber-body links,
// System::apply_matvec / ::apply_preconditioner and the RHS of the mobility system on whole solution vectors -- on one
// device (skb_flow_*) and on a group member (skb_flow_group_*, which skb_mflow drives on its members) -- and the
// refusals they share.  Built on the matvec orchestration of skb_matvec.cu.
#include "skb_flow.hpp"

#include <algorithm>
#include <cmath>
#include <vector>

using namespace skb;

void skb::split_forces_torques(const double *ft, int n_bodies, std::vector<double> &f, std::vector<double> &t) {
    f.resize(3 * (size_t)n_bodies);
    t.resize(3 * (size_t)n_bodies);
    for (int b = 0; b < n_bodies; ++b)
        for (int k = 0; k < 3; ++k) {
            f[3 * b + k] = ft[6 * b + k];     // forces_torques.block(0,0,3,n)  body_container.cpp:134
            t[3 * b + k] = ft[6 * b + 3 + k]; // forces_torques.block(3,0,3,n)
        }
}

// ---- the whole-vector operator and preconditioner with the bodies on the device (skb_body.cu) -------------------
// The solution vector is [fibers (4 per node) | shell (3 per node) | bodies (3 n_b + 6 each)] (get_solution_maps,
// system.cpp:69-92); single device, whole target list.

extern "C" {

int skb_flow_set_body_operators(skb_flow *fl, const int *n_nodes, int n_bodies, const double *node_weights,
                                const double *ex, const double *ey, const double *ez, const double *A_inv) {
    const char *who = "skb_flow_set_body_operators";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (fl->grp.member())
        return set_error(SKB_ERR_INVALID, "%s: the body block runs on a single device, not in a group", who);
    if (n_bodies != fl->n_bodies)
        return set_error(SKB_ERR_INVALID, "%s: %d bodies, skb_flow_set_bodies has %d", who, n_bodies, fl->n_bodies);
    if (n_bodies > 0 && (!n_nodes || !node_weights || !ex || !ey || !ez))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    CUDA_TRY(cudaSetDevice(fl->dev));
    return fl->bodies.set_operators(n_nodes, n_bodies, fl->n_body, fl->h_r_body.data(), fl->h_centers.data(),
                                    node_weights, ex, ey, ez, A_inv, fl->stream);
}

int skb_flow_set_fiber_links(skb_flow *fl, const int *body, const double *site, const double *bending_rigidity) {
    const char *who = "skb_flow_set_fiber_links";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (fl->grp.member())
        return set_error(SKB_ERR_INVALID, "%s: the body block runs on a single device, not in a group", who);
    if (body && fl->n_fibers > 0 && (!site || !bending_rigidity))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    CUDA_TRY(cudaSetDevice(fl->dev));
    return fl->bodies.set_links(all_fibers(fl), fl->ops, fl->n_bodies, fl->h_centers.data(), body, site,
                                bending_rigidity, fl->stream);
}

} // extern "C"

// ---- rigid bodies placed from their body frame (BodyOps::set_frames / ::place, DESIGN.md §3.6) --------------------

void skb::quaternion_rotation(const double *q, double *R) {
    const double w = q[0], x = q[1], y = q[2], z = q[3];
    const double tx = 2.0 * x, ty = 2.0 * y, tz = 2.0 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1.0 - (tyy + tzz), R[1] = txy - twz, R[2] = txz + twy;
    R[3] = txy + twz, R[4] = 1.0 - (txx + tzz), R[5] = tyz - twx;
    R[6] = txz - twy, R[7] = tyz + twx, R[8] = 1.0 - (txx + tyy);
}

// the body rows [lo, hi) whose frames and operators the flow keeps: a group member's own, else every row (hi < 0); then
// the flow's device is current
static int body_window(skb_flow *fl, long long &lo, long long &hi) {
    lo = 0;
    hi = -1;
    CUDA_TRY(cudaSetDevice(fl->dev));
    if (fl->grp.member()) {
        SKB_TRY(prepare_matvec_targets(fl));
        lo = fl->ba;
        hi = fl->bb;
    }
    return SKB_OK;
}

// the frames of the flow's bodies (a member: for its body rows)
static int body_frames(skb_flow *fl, const char *who, const int *n_nodes, int n_bodies, const double *pos_ref,
                       const double *normal_ref, const double *node_weights, const double *ex0, const double *ey0,
                       const double *ez0, const double *A_inv0) {
    long long lo, hi;
    SKB_TRY(body_window(fl, lo, hi));
    if (n_bodies != fl->n_bodies)
        return set_error(SKB_ERR_INVALID, "%s: %d bodies, skb_flow_set_bodies has %d", who, n_bodies, fl->n_bodies);
    if (n_bodies > 0 && (!n_nodes || !pos_ref || !normal_ref || !node_weights || !ex0 || !ey0 || !ez0))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    return fl->bodies.set_frames(n_nodes, n_bodies, fl->n_body, pos_ref, normal_ref, node_weights, ex0, ey0, ez0,
                                 A_inv0, fl->stream, lo, hi);
}

// frames that match the flow's bodies and its body rows, finite unit quaternions
int skb::placement_args(skb_flow *fl, const char *who, const double *centers, const double *orientations,
                        std::vector<double> &R) {
    long long lo, hi;
    SKB_TRY(body_window(fl, lo, hi));
    const BodyOps &b = fl->bodies;
    if (!b.has_frames())
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_body_frames first", who);
    if (b.frame_bodies() != fl->n_bodies || b.frame_nodes() != fl->n_body)
        return set_error(SKB_ERR_INVALID, "%s: the flow has %d bodies of %lld nodes, the frames %d bodies of %lld nodes "
                                          "(set the frames again after skb_flow_set_bodies changes them)", who,
                         fl->n_bodies, fl->n_body, b.frame_bodies(), b.frame_nodes());
    if (!b.frame_window(lo, hi))
        return set_error(SKB_ERR_INVALID, "%s: the body rows changed since the frames were set (set them again)", who);
    const int nb = fl->n_bodies;
    if (nb > 0 && (!centers || !orientations))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    R.resize((size_t)nb * 9);
    for (int i = 0; i < nb; ++i) {
        const double *q = orientations + 4 * (size_t)i;
        const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
        if (!(std::fabs(n2 - 1.0) <= SKB_UNIT_QUATERNION_TOL))
            return set_error(SKB_ERR_INVALID, "%s: orientation %d = (%g, %g, %g, %g) is not a finite unit quaternion "
                                              "(|q|^2 - 1 = %g, tolerance %g)", who, i, q[0], q[1], q[2], q[3],
                             n2 - 1.0, SKB_UNIT_QUATERNION_TOL);
        quaternion_rotation(q, &R[9 * (size_t)i]);
    }
    return SKB_OK;
}

// after placement_args: the nodes and normals through skb_flow_set_bodies (which drops the operators and the links),
// then the operators from the frames
static int place_bodies(skb_flow *fl, const double *centers, const double *orientations, const std::vector<double> &R) {
    std::vector<double> pos, nrm;
    fl->bodies.placed_geometry(R.data(), centers, pos, nrm);
    SKB_TRY(skb_flow_set_bodies(fl, pos.data(), nrm.data(), fl->n_body, centers, fl->n_bodies));
    CUDA_TRY(cudaSetDevice(fl->dev));
    SKB_TRY(fl->bodies.place(R.data(), fl->h_r_body.data(), fl->h_centers.data(), fl->stream));
    fl->h_orient.assign(orientations, orientations + 4 * (size_t)fl->n_bodies);
    fl->placed = true;
    return SKB_OK;
}

extern "C" {

int skb_flow_set_body_frames(skb_flow *fl, const int *n_nodes, int n_bodies, const double *node_pos_ref,
                             const double *node_normal_ref, const double *node_weights, const double *ex0,
                             const double *ey0, const double *ez0, const double *A_inv0) {
    const char *who = "skb_flow_set_body_frames";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (fl->grp.member())
        return set_error(SKB_ERR_INVALID, "%s: a group member sets its frames with skb_flow_group_set_body_frames", who);
    return body_frames(fl, who, n_nodes, n_bodies, node_pos_ref, node_normal_ref, node_weights, ex0, ey0, ez0, A_inv0);
}

int skb_flow_place_bodies(skb_flow *fl, const double *centers, const double *orientations) {
    const char *who = "skb_flow_place_bodies";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (fl->grp.member())
        return set_error(SKB_ERR_INVALID, "%s: a group member places its bodies with skb_flow_group_place_bodies", who);
    std::vector<double> R;
    SKB_TRY(placement_args(fl, who, centers, orientations, R));
    return place_bodies(fl, centers, orientations, R);
}

int skb_flow_get_body_operators(skb_flow *fl, double *ex, double *ey, double *ez, double *A_inv) {
    const char *who = "skb_flow_get_body_operators";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (fl->n_bodies > 0 && !fl->bodies.has_operators())
        return set_error(SKB_ERR_INVALID, "%s: no body operators are resident (skb_flow_set_body_operators or "
                                          "skb_flow_place_bodies after skb_flow_set_bodies)", who);
    if (fl->n_bodies > 0 && A_inv && !fl->bodies.has_inverse())
        return set_error(SKB_ERR_INVALID, "%s: the resident body operators have no A_inv", who);
    if (fl->n_bodies == 0)
        return SKB_OK;
    CUDA_TRY(cudaSetDevice(fl->dev));
    return fl->bodies.read(ex, ey, ez, A_inv, fl->stream);
}

} // extern "C"

// ---- the per-fiber dense operators (FiberOps, skb_fiber.cu): their class tables, their upload or device build, the
// fibers' RHS and the three GEMVs on the own fibers --------------------------------------------------------------

// frame of the fiber operators' GEMV entry points: the operators' check (`inverse`: with their inverse), nothing to do
// without own fibers, the arguments, then call(nodes of the own fibers) on the flow's device
template <class Call> static int fiber_ops_call(skb_flow *fl, const char *who, bool inverse, bool args, Call call) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    SKB_TRY(fl->ops.ready(who, inverse));
    begin_stats(fl);
    if (fl->ops.empty())
        return SKB_OK;
    if (!args)
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    CUDA_TRY(cudaSetDevice(fl->dev));
    return call((size_t)(fl->fb - fl->fa));
}

extern "C" {

int skb_flow_set_fiber_class(skb_flow *fl, int n_nodes, const double *D_1_0, const double *P_downsample_bc) {
    if (!fl || !D_1_0 || !P_downsample_bc)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_fiber_class: NULL argument");
    CUDA_TRY(cudaSetDevice(fl->dev));
    fl->bodies.drop_links(); // a new node count moves the class table's offsets the links hold
    return fl->ops.set_class(n_nodes, D_1_0, P_downsample_bc, fl->stream);
}

int skb_flow_set_fiber_class_derivatives(skb_flow *fl, int n_nodes, const double *D_2_0, const double *D_3_0,
                                         const double *D_4_0) {
    if (!fl || !D_2_0 || !D_3_0 || !D_4_0)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_fiber_class_derivatives: NULL argument");
    CUDA_TRY(cudaSetDevice(fl->dev));
    return fl->ops.set_class_derivatives(n_nodes, D_2_0, D_3_0, D_4_0, fl->stream);
}

int skb_flow_set_fiber_operators(skb_flow *fl, const double *A, const double *force_operator, const double *xs,
                                 const double *length_prev, const int *plus_bc_velocity) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_fiber_operators: NULL flow");
    fl->ops.invalidate();
    CUDA_TRY(cudaSetDevice(fl->dev));
    OwnFibers own;
    SKB_TRY(own_fibers(fl, "skb_flow_set_fiber_operators", own));
    if (own.count() > 0 && (!A || !force_operator || !xs || !length_prev || !plus_bc_velocity))
        return set_error(SKB_ERR_INVALID, "skb_flow_set_fiber_operators: NULL argument");
    return fl->ops.upload(own, A, force_operator, xs, length_prev, plus_bc_velocity);
}

int skb_flow_set_fiber_preconditioner(skb_flow *fl, const double *A_inv) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_fiber_preconditioner: NULL flow");
    CUDA_TRY(cudaSetDevice(fl->dev));
    return fl->ops.upload_inverse(A_inv, fl->stream);
}

int skb_flow_build_fiber_operators(skb_flow *fl, const skb_fiber_params *params, double dt, double eta) {
    const char *who = "skb_flow_build_fiber_operators";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    fl->ops.invalidate();
    if (!(dt > 0) || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "%s: dt = %g, eta = %g (both must be > 0)", who, dt, eta);
    CUDA_TRY(cudaSetDevice(fl->dev));
    OwnFibers own;
    SKB_TRY(own_fibers(fl, who, own));
    if (own.count() > 0 && !params)
        return set_error(SKB_ERR_INVALID, "%s: NULL params", who);
    // device_ms spans the assembly and inverse kernels, total_ms also the table uploads before them
    return fl->ops.build(own, params, dt, eta, &fl->launches,
                         [&](const FiberOps::Step &stage, const FiberOps::Step &launch) {
                             begin_stats(fl);
                             return host_frame(fl, stage, launch, nothing);
                         });
}

// checks shared by the two forms of the fiber RHS, then the own fibers on the flow's device; stats of no launch
static int fiber_rhs_args(skb_flow *fl, const char *who, const skb_fiber_params *params, const double *rhs, double dt,
                          double eta, OwnFibers &own) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (!(dt > 0) || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "%s: dt = %g, eta = %g (both must be > 0)", who, dt, eta);
    CUDA_TRY(cudaSetDevice(fl->dev));
    SKB_TRY(own_fibers(fl, who, own));
    if (own.count() > 0 && (!params || !rhs))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    begin_stats(fl);
    return device_stats(fl);
}

int skb_flow_build_fiber_rhs(skb_flow *fl, const skb_fiber_params *params, const double *v_growth,
                             const double *force_scale, const double *v_on_fibers, const double *f_external, double dt,
                             double eta, double *rhs) {
    OwnFibers own;
    SKB_TRY(fiber_rhs_args(fl, "skb_flow_build_fiber_rhs", params, rhs, dt, eta, own));
    const long long nf = own.nodes();
    // staged here, so that the kernel's arguments are known before its frame (host_call keeps them); device_ms spans
    // the kernel, total_ms also the uploads and the tables' stage before it and the download after it
    Transfers xfer{{up(v_on_fibers, 3 * nf), up(f_external, 3 * nf)}, {down(rhs, 4 * nf)}};
    SKB_TRY(stage_slots(fl->slots, xfer));
    return fl->ops.rhs(own, params, v_growth, force_scale, v_on_fibers ? xfer.up[0].dev : nullptr,
                       f_external ? xfer.up[1].dev : nullptr, dt, eta, xfer.down[0].dev, &fl->launches,
                       [&](const FiberOps::Step &stage, const FiberOps::Step &launch) {
                           return host_call(fl, xfer, [&](const Transfers &) { return launch(); }, stage);
                       });
}

int skb_flow_build_fiber_rhs_device(skb_flow *fl, const skb_fiber_params *params, const double *v_growth,
                                    const double *force_scale, const double *d_v_on_fibers, const double *d_f_external,
                                    double dt, double eta, double *d_rhs, void *stream) {
    OwnFibers own;
    SKB_TRY(fiber_rhs_args(fl, "skb_flow_build_fiber_rhs_device", params, d_rhs, dt, eta, own));
    own.stream = (cudaStream_t)stream;
    return fl->ops.rhs(own, params, v_growth, force_scale, d_v_on_fibers, d_f_external, dt, eta, d_rhs, &fl->launches,
                       [&](const FiberOps::Step &stage, const FiberOps::Step &launch) {
                           return device_frame(fl, stream, [&]() -> int {
                               SKB_TRY(stage());
                               return launch();
                           });
                       });
}

int skb_flow_get_fiber_operators(skb_flow *fl, double *A, double *force_operator, double *xs, double *A_inv) {
    const char *who = "skb_flow_get_fiber_operators";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    SKB_TRY(fl->ops.ready(who, A_inv != nullptr));
    CUDA_TRY(cudaSetDevice(fl->dev));
    return fl->ops.read(A, force_operator, xs, A_inv, fl->stream);
}

// host pointers: through host_frame on the flow's stream; device pointers: asynchronously on the caller's stream
int skb_flow_apply_fiber_preconditioner(skb_flow *fl, const double *x_fibers, double *y) {
    return fiber_ops_call(fl, "skb_flow_apply_fiber_preconditioner", true, x_fibers && y, [&](size_t nf) {
        Transfers xfer{{up(x_fibers, 4 * nf)}, {down(y, 4 * nf)}};
        return host_call(fl, xfer, [&](const Transfers &io) {
            return fl->ops.precondition(io.up[0].dev, io.down[0].dev, fl->cur, &fl->launches);
        });
    });
}

int skb_flow_apply_fiber_preconditioner_device(skb_flow *fl, const double *d_x_fibers, double *d_y, void *stream) {
    return fiber_ops_call(fl, "skb_flow_apply_fiber_preconditioner_device", true, d_x_fibers && d_y, [&](size_t) {
        return device_frame(fl, stream,
                            [&] { return fl->ops.precondition(d_x_fibers, d_y, fl->cur, &fl->launches); });
    });
}

int skb_flow_apply_fiber_force(skb_flow *fl, const double *x_fibers, double *fw) {
    return fiber_ops_call(fl, "skb_flow_apply_fiber_force", false, x_fibers && fw, [&](size_t nf) {
        Transfers xfer{{up(x_fibers, 4 * nf)}, {down(fw, 3 * nf)}};
        return host_call(fl, xfer, [&](const Transfers &io) {
            return fl->ops.force(io.up[0].dev, io.down[0].dev, fl->cur, &fl->launches);
        });
    });
}

int skb_flow_fiber_matvec(skb_flow *fl, const double *x_fibers, const double *v_fibers, const double *v_fib_boundary,
                          double *res) {
    return fiber_ops_call(fl, "skb_flow_fiber_matvec", false, x_fibers && v_fibers && res, [&](size_t nf) {
        Transfers xfer{{up(x_fibers, 4 * nf), up(v_fibers, 3 * nf), up(v_fib_boundary, 7LL * fl->ops.n_fibers())},
                       {down(res, 4 * nf)}};
        return host_call(fl, xfer, [&](const Transfers &io) {
            return fl->ops.matvec(io.up[0].dev, io.up[1].dev, v_fib_boundary ? io.up[2].dev : nullptr, io.down[0].dev,
                                  fl->cur, &fl->launches);
        });
    });
}

int skb_flow_apply_fiber_force_device(skb_flow *fl, const double *d_x_fibers, double *d_fw, void *stream) {
    return fiber_ops_call(fl, "skb_flow_apply_fiber_force_device", false, d_x_fibers && d_fw, [&](size_t) {
        return device_frame(fl, stream, [&] { return fl->ops.force(d_x_fibers, d_fw, fl->cur, &fl->launches); });
    });
}

int skb_flow_fiber_matvec_device(skb_flow *fl, const double *d_x_fibers, const double *d_v_fibers,
                                 const double *d_v_fib_boundary, double *d_res, void *stream) {
    return fiber_ops_call(fl, "skb_flow_fiber_matvec_device", false, d_x_fibers && d_v_fibers && d_res, [&](size_t) {
        return device_frame(fl, stream, [&] {
            return fl->ops.matvec(d_x_fibers, d_v_fibers, d_v_fib_boundary, d_res, fl->cur, &fl->launches);
        });
    });
}

} // extern "C"

// ---- the refusals of the system calls, of every family ----

int skb::system_ready(skb_flow *fl, const char *who, const Calls &calls, bool precondition, bool step) {
    if (fl->n_fibers > 0 && !step) // no fibers: the empty operator set, uploaded or not
        SKB_TRY(fl->ops.ready(who, precondition));
    if (fl->n_bodies == 0)
        return SKB_OK;
    if (step && (!fl->bodies.has_frames() || !fl->placed || !fl->bodies.has_operators()))
        return set_error(SKB_ERR_INVALID, "%s: the step places the bodies from their frames: call %sset_body_frames "
                                          "and a first %splace_bodies", who, calls.setup, calls.setup);
    if (!fl->bodies.has_operators())
        return set_error(SKB_ERR_INVALID, "%s: call %sset_body_operators after %sset_bodies", who, calls.setup,
                         calls.geometry);
    if (precondition && !fl->bodies.has_inverse())
        return set_error(SKB_ERR_INVALID, "%s: %sset_body_%s was given no A_inv", who, calls.setup,
                         step ? "frames" : "operators");
    if (!precondition && fl->n_fibers > 0 && !fl->bodies.has_links())
        return set_error(SKB_ERR_INVALID, "%s: call %sset_fiber_links after %sset_fibers / %sset_bodies (NULL body: no "
                                          "fiber is bound)", who, calls.setup, calls.geometry, calls.geometry);
    return SKB_OK;
}

int skb::dense_rows(skb_flow *fl, skb_dense *dn, const char *who, bool precondition) {
    const char *op_name = precondition ? "M_inv" : "stresslet_plus_complementary";
    if (!dn)
        return set_error(SKB_ERR_INVALID, "%s: the periphery rows need their rows of %s (dn == NULL)", who, op_name);
    SKB_TRY(prepare_matvec_targets(fl));
    int dn_dev = -1;
    int64_t rows = -1, cols = -1;
    SKB_TRY(skb_dense_device(dn, 0, &dn_dev));
    SKB_TRY(skb_dense_shape(dn, precondition ? SKB_DENSE_M_INV : SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY, &rows, &cols));
    const long long n_sw = fl->sb - fl->sa;
    if (dn_dev != fl->dev || rows != 3 * n_sw || cols != 3 * fl->n_shell)
        return set_error(SKB_ERR_INVALID, "%s: the dense handle holds a %lld x %lld %s on device %d, need the flow's "
                                          "%lld own rows x %lld of the %lld periphery nodes on device %d", who,
                         (long long)rows, (long long)cols, op_name, dn_dev, 3 * n_sw, 3 * fl->n_shell, fl->n_shell,
                         fl->dev);
    return SKB_OK;
}

int skb::whole_targets(skb_flow *fl, const char *who, const char *hint) {
    SKB_TRY(prepare_matvec_targets(fl));
    const long long n_all = fl->n_fib + fl->n_shell + fl->n_body;
    if (fl->n_win != n_all)
        return set_error(SKB_ERR_INVALID, "%s: needs the whole target list (%lld of %lld rows are set by a target window "
                                          "or ranges)%s", who, fl->n_win, n_all, hint);
    return SKB_OK;
}

int skb::system_args(skb_flow *fl, skb_dense *dn, const char *who, bool precondition, bool args) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (fl->grp.member())
        return set_error(SKB_ERR_INVALID, "%s: multi-GPU is not supported: a body's K^T lambda needs all of its nodes "
                                          "(the reference keeps the bodies on rank 0); use a single-device flow", who);
    CUDA_TRY(cudaSetDevice(fl->dev));
    SKB_TRY(whole_targets(fl, who, "; multi-GPU is not supported"));
    if (fl->n_shell > 0)
        SKB_TRY(dense_rows(fl, dn, who, precondition));
    SKB_TRY(system_ready(fl, who, kFlowCalls, precondition));
    if (!args)
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    begin_stats(fl);
    return SKB_OK;
}

long long skb::solution_size(const skb_flow *fl) {
    return 4 * fl->n_fib + 3 * fl->n_shell + (fl->n_bodies > 0 ? fl->bodies.solution_size() : 0);
}

// System::apply_matvec (system.cpp:269-324) on fl->cur: the links, forces / torques and densities of the bodies from
// x, then apply_matvec_core unchanged, then bc.matvec on its v_bodies rows
static int system_matvec_core(skb_flow *fl, skb_dense *dn, const double *d_x, double eta, double *d_res) {
    const long long nf = fl->n_fib, ns = fl->n_shell;
    const double *x_fib = d_x, *x_shell = d_x + 4 * nf, *x_bodies = x_shell + 3 * ns;
    double *res_fib = d_res, *res_shell = d_res + 4 * nf, *res_bodies = res_shell + 3 * ns;
    const double *link = nullptr, *bd = nullptr, *f = nullptr, *t = nullptr;
    if (fl->n_bodies > 0) { // fc.calculate_link_conditions (system.cpp:311), the densities out of x_bodies
        SKB_TRY(fl->bodies.links(fl->ops, (const double *)fl->fiber_length.ptr, x_fib, x_bodies, &link, fl->cur,
                                 &fl->launches));
        bd = fl->bodies.densities();
        f = fl->bodies.forces();
        t = fl->bodies.torques();
    }
    SKB_TRY(fl->tmp_b.ensure((size_t)fl->n_body * 24 + 8));
    double *v_bodies = (double *)fl->tmp_b.ptr;
    SKB_TRY(apply_matvec_core(fl, dn, x_fib, x_shell, bd, f, t, link, eta, res_fib, res_shell, v_bodies));
    // res_bodies = bc.matvec(v_bodies, x_bodies)                          system.cpp:320
    return fl->n_bodies > 0 ? fl->bodies.matvec(x_bodies, v_bodies, res_bodies, fl->cur, &fl->launches) : SKB_OK;
}

// System::apply_preconditioner (system.cpp:248-262) on fl->cur
static int system_precondition_core(skb_flow *fl, skb_dense *dn, const double *d_x, double *d_y) {
    const long long nf = fl->n_fib, ns = fl->n_shell;
    SKB_TRY(fl->ops.precondition(d_x, d_y, fl->cur, &fl->launches));
    if (ns > 0) {
        SKB_TRY(skb_dense_apply_device(dn, SKB_DENSE_M_INV, d_x + 4 * nf, nullptr, d_y + 4 * nf, fl->cur));
        fl->launches += 1;
    }
    return fl->n_bodies > 0
               ? fl->bodies.precondition(d_x + 4 * nf + 3 * ns, d_y + 4 * nf + 3 * ns, fl->cur, &fl->launches)
               : SKB_OK;
}

extern "C" {

int skb_flow_apply_system_matvec(skb_flow *fl, skb_dense *dn, const double *x, double eta, double *res) {
    const char *who = "skb_flow_apply_system_matvec";
    SKB_TRY(system_args(fl, dn, who, false, (x && res) || solution_size(fl) == 0));
    if (!(eta > 0))
        return set_error(SKB_ERR_INVALID, "%s: eta = %g", who, eta);
    const size_t n = (size_t)solution_size(fl);
    if (n == 0)
        return SKB_OK;
    Transfers xfer{{up(x, n)}, {down(res, n)}};
    return host_call(fl, xfer, [&](const Transfers &io) {
        return system_matvec_core(fl, dn, io.up[0].dev, eta, io.down[0].dev);
    });
}

int skb_flow_apply_system_matvec_device(skb_flow *fl, skb_dense *dn, const double *d_x, double eta, double *d_res,
                                        void *stream) {
    const char *who = "skb_flow_apply_system_matvec_device";
    SKB_TRY(system_args(fl, dn, who, false, (d_x && d_res) || solution_size(fl) == 0));
    if (!(eta > 0))
        return set_error(SKB_ERR_INVALID, "%s: eta = %g", who, eta);
    if (solution_size(fl) == 0)
        return SKB_OK;
    return device_frame(fl, stream, [&] { return system_matvec_core(fl, dn, d_x, eta, d_res); });
}

int skb_flow_apply_system_preconditioner(skb_flow *fl, skb_dense *dn, const double *x, double *y) {
    const char *who = "skb_flow_apply_system_preconditioner";
    SKB_TRY(system_args(fl, dn, who, true, (x && y) || solution_size(fl) == 0));
    const size_t n = (size_t)solution_size(fl);
    if (n == 0)
        return SKB_OK;
    Transfers xfer{{up(x, n)}, {down(y, n)}};
    return host_call(fl, xfer,
                     [&](const Transfers &io) { return system_precondition_core(fl, dn, io.up[0].dev, io.down[0].dev); });
}

int skb_flow_apply_system_preconditioner_device(skb_flow *fl, skb_dense *dn, const double *d_x, double *d_y,
                                                void *stream) {
    const char *who = "skb_flow_apply_system_preconditioner_device";
    SKB_TRY(system_args(fl, dn, who, true, (d_x && d_y) || solution_size(fl) == 0));
    if (solution_size(fl) == 0)
        return SKB_OK;
    return device_frame(fl, stream, [&] { return system_precondition_core(fl, dn, d_x, d_y); });
}

} // extern "C"

// ---- the right-hand side of the whole system (System::prep_state_for_solver, system.cpp:398-458) --------------------
// One device call from the external forces to the RHS vector [fibers | shell | bodies], laid out as Solver::set_RHS
// copies it (solver_hydro.cpp:51-61).  Its flow is matvec_core unchanged -- f_ext as the fiber strengths, zero periphery
// and body densities, the bodies' external F_T -- so that the symmetric and cross kernels, the self term and, in a
// group, the exchange through the window serve it as they serve the matvec.

// the zero densities of the RHS flow (and the zero forces it takes for an absent f_external or F_T), the velocities,
// and the kernels the call launches besides matvec_core's, loaded now (the first launch of a group member must not load
// a kernel lazily while a peer on the same device spins on a flag)
static int rhs_buffers(skb_flow *fl) {
    const long long n = std::max<long long>({3 * (fl->fb - fl->fa), 3 * (fl->sb - fl->sa), 3 * fl->n_body,
                                             3LL * fl->n_bodies, 1LL});
    SKB_TRY(fl->zeros.ensure((size_t)n * 8));
    fl->n_zeros = n;
    SKB_TRY(fl->vel.ensure((size_t)fl->n_win * 24 + 8));
    SKB_TRY(load_source_kernels());
    return load_rhs_rows_kernel();
}

// System::prep_state_for_solver's RHS (system.cpp:421-455) on fl->cur, the rows of this flow's target list: d_fext 3 per
// own fiber node or NULL (no external fiber force), d_f / d_t 3 per body, complete, or NULL (zero); d_rhs_fib 4 per own
// fiber node, d_rhs_shell 3 per own periphery row, d_rhs_bodies in the x_bodies layout (the rows BodyOps owns written).
// params / v_growth / force_scale per own fiber.  Every check, the fiber block's included, precedes the first launch.
static int system_rhs_core(skb_flow *fl, OwnFibers own, const skb_fiber_params *params, const double *v_growth,
                           const double *force_scale, const double *d_fext, const double *d_f, const double *d_t,
                           double dt, double eta, double *d_rhs_fib, double *d_rhs_shell, double *d_rhs_bodies) {
    const long long n_fw = fl->fb - fl->fa, n_sw = fl->sb - fl->sa;
    double *d_v = (double *)fl->vel.ptr;
    const double *zero = (const double *)fl->zeros.ptr;
    own.stream = fl->cur;
    fl->bg.dn = nullptr; // no dense operator: nothing goes to the background streamer
    fl->bg.launched = false;
    auto run = [&](const FiberOps::Step *stage, const FiberOps::Step *launch) -> int {
        if (stage) // the fiber block's per-fiber tables
            SKB_TRY((*stage)());
        CUDA_TRY(cudaMemsetAsync(fl->zeros.ptr, 0, (size_t)fl->n_zeros * 8, fl->cur));
        // v_all = fc.flow(r_all, f_ext, eta), self term subtracted (system.cpp:425), + bc.flow(r_all, 0, F_T, eta)
        // (:442).  F_T are complete on every member and go straight to the body flow (no ft_exchange): each counts once
        SKB_TRY(matvec_core(fl, d_fext ? d_fext : zero, zero, zero, d_f ? d_f : zero, d_t ? d_t : zero, eta, d_v));
        // v_all += psc.flow + bs.flow (:445-446).  The body evaluator's matvec targets are the rows of d_v, in its order
        SKB_TRY(add_sources(fl, (const double *)fl->body[1].r_trg.ptr, fl->n_win, eta, d_v, fl->cur));
        // fc.update_rhs(dt, v_fibers, motor + f_ext) + fc.apply_bcs(dt, v_fibers, f_ext) (:451-453)
        if (launch)
            SKB_TRY((*launch)());
        // bc.update_RHS(v_bodies), shell.update_RHS(v_shell) (:448, 455)
        return fl->bodies.rhs_rows(fl->n_bodies > 0, d_v + 3 * (n_fw + n_sw), d_rhs_bodies, d_v + 3 * n_fw, n_sw,
                                   d_rhs_shell, fl->cur, &fl->launches);
    };
    bool framed = false; // FiberOps::rhs calls the frame only when there are own fibers
    SKB_TRY(fl->ops.rhs(own, params, v_growth, force_scale, d_v, d_fext, dt, eta, d_rhs_fib, &fl->launches,
                        [&](const FiberOps::Step &stage, const FiberOps::Step &launch) {
                            framed = true;
                            return run(&stage, &launch);
                        }));
    return framed ? SKB_OK : run(nullptr, nullptr);
}

static int finite(const double *a, size_t n) {
    for (size_t i = 0; i < n; ++i)
        if (!std::isfinite(a[i]))
            return 0;
    return 1;
}

// the refusals of the two skb_flow forms, before any launch; then the own fibers, the flow's device current, the
// buffers sized
static int system_rhs_args(skb_flow *fl, const char *who, const skb_fiber_params *params, bool out, double dt,
                           double eta, OwnFibers &own) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (fl->grp.member())
        return set_error(SKB_ERR_INVALID, "%s: a group member's rows need the others' fiber forces; over several devices "
                                          "use skb_mflow_build_system_rhs", who);
    if (!(dt > 0) || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "%s: dt = %g, eta = %g (both must be > 0)", who, dt, eta);
    CUDA_TRY(cudaSetDevice(fl->dev));
    SKB_TRY(own_fibers(fl, who, own));
    SKB_TRY(whole_targets(fl, who, "; over several devices use skb_mflow_build_system_rhs"));
    if (fl->n_bodies > 0 && !fl->bodies.has_operators())
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_set_body_operators after skb_flow_set_bodies (the body rows "
                                          "are laid out by its node counts)", who);
    if ((own.count() > 0 && !params) || (solution_size(fl) > 0 && !out))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    begin_stats(fl);
    return rhs_buffers(fl);
}

extern "C" {

int skb_flow_build_system_rhs(skb_flow *fl, const skb_fiber_params *params, const double *v_growth,
                              const double *force_scale, const double *f_external, const double *body_forces_torques,
                              double dt, double eta, double *rhs) {
    const char *who = "skb_flow_build_system_rhs";
    OwnFibers own;
    SKB_TRY(system_rhs_args(fl, who, params, rhs != nullptr, dt, eta, own));
    const long long nf = fl->n_fib, ns = fl->n_shell;
    if ((f_external && !finite(f_external, (size_t)nf * 3)) ||
        (body_forces_torques && !finite(body_forces_torques, (size_t)fl->n_bodies * 6)))
        return set_error(SKB_ERR_INVALID, "%s: a non-finite external force or torque", who);
    const size_t n = (size_t)solution_size(fl);
    if (n == 0)
        return SKB_OK;
    std::vector<double> f, t;
    if (body_forces_torques && fl->n_bodies > 0)
        split_forces_torques(body_forces_torques, fl->n_bodies, f, t);
    Transfers xfer{{up(f_external, 3 * nf), up(f.data(), f.size()), up(t.data(), t.size())}, {down(rhs, n)}};
    return host_call(fl, xfer, [&](const Transfers &io) {
        double *d_rhs = io.down[0].dev;
        return system_rhs_core(fl, own, params, v_growth, force_scale, f_external && nf ? io.up[0].dev : nullptr,
                               f.empty() ? nullptr : io.up[1].dev, t.empty() ? nullptr : io.up[2].dev, dt, eta, d_rhs,
                               d_rhs + 4 * nf, d_rhs + 4 * nf + 3 * ns);
    });
}

int skb_flow_build_system_rhs_device(skb_flow *fl, const skb_fiber_params *params, const double *v_growth,
                                     const double *force_scale, const double *d_f_external,
                                     const double *d_body_forces, const double *d_body_torques, double dt, double eta,
                                     double *d_rhs, void *stream) {
    OwnFibers own;
    SKB_TRY(system_rhs_args(fl, "skb_flow_build_system_rhs_device", params, d_rhs != nullptr, dt, eta, own));
    if (solution_size(fl) == 0)
        return SKB_OK;
    const long long nf = fl->n_fib, ns = fl->n_shell;
    return device_frame(fl, stream, [&] {
        return system_rhs_core(fl, own, params, v_growth, force_scale, nf ? d_f_external : nullptr,
                               fl->n_bodies ? d_body_forces : nullptr, fl->n_bodies ? d_body_torques : nullptr, dt, eta,
                               d_rhs, d_rhs + 4 * nf, d_rhs + 4 * nf + 3 * ns);
    });
}

} // extern "C"

// a group member's: the links of the own fibers, apply_matvec_core with the exchange of their partial forces, the owned
// body rows; on fl->cur
static int member_system_matvec_core(skb_flow *fl, skb_dense *dn, const double *d_x_fib, const double *d_x_shell,
                                     const double *d_x_bodies, double eta, double *d_res_fib, double *d_res_shell,
                                     double *d_res_bodies) {
    const double *link = nullptr, *bd = nullptr, *f = nullptr, *t = nullptr;
    if (fl->n_bodies > 0) { // the links of the own fibers; their partial forces / torques on every body
        const auto &off = fl->h_fiber_off;
        const long long f0 = fl->n_fibers ? std::lower_bound(off.begin(), off.end(), fl->fa) - off.begin() : 0;
        SKB_TRY(fl->bodies.links(fl->ops, (const double *)fl->fiber_length.ptr + f0, d_x_fib, d_x_bodies, &link,
                                 fl->cur, &fl->launches));
        bd = fl->bodies.densities();
        f = fl->bodies.forces();
        t = fl->bodies.torques();
    }
    double *v_bodies = (double *)fl->tmp_b.ptr; // own body rows
    fl->ft_exchange = true;
    const int rc = apply_matvec_core(fl, dn, d_x_fib, d_x_shell, bd, f, t, link, eta, d_res_fib, d_res_shell, v_bodies);
    fl->ft_exchange = false;
    SKB_TRY(rc);
    return fl->n_bodies > 0 ? fl->bodies.matvec(d_x_bodies, v_bodies, d_res_bodies, fl->cur, &fl->launches) : SKB_OK;
}

// a member's slice of a per-fiber array of ALL fibers (NULL stays NULL, and so does the slice of no fibers)
template <class T> static const T *own_slice(const T *all, const OwnFibers &own) {
    return all && own.count() > 0 ? all + own.f0 : nullptr;
}

int skb::flow_member_rhs_prepare(skb_flow *fl, const skb_fiber_params *params, const double *v_growth,
                                 const double *force_scale, double dt, double eta) {
    const char *who = "skb_mflow_build_system_rhs";
    CUDA_TRY(cudaSetDevice(fl->dev));
    OwnFibers own;
    SKB_TRY(own_fibers(fl, who, own));
    if (fl->n_bodies > 0 && !fl->bodies.has_operators())
        return set_error(SKB_ERR_INVALID, "%s: call skb_mflow_set_body_operators after skb_mflow_set_bodies", who);
    SKB_TRY(rhs_buffers(fl));
    // the fiber block's checks, and its tables uploaded once so that their buffers have their size before any launch
    return fl->ops.rhs(own, own_slice(params, own), own_slice(v_growth, own), own_slice(force_scale, own), nullptr,
                       nullptr, dt, eta, nullptr, &fl->launches,
                       [&](const FiberOps::Step &stage, const FiberOps::Step &) -> int {
                           SKB_TRY(stage());
                           CUDA_TRY(cudaStreamSynchronize(own.stream));
                           return SKB_OK;
                       });
}

// ---- the whole-vector calls of a rank-per-GPU group member (skb_flow_group_*, include/skelly_b200_flow.h) ----------
// A member holds only its own rows of the solution vector, in ascending global order (distributed.system_rows):
// x_local = [4 per own fiber node | 3 per own periphery row | own body rows].  Before a matvec or a preconditioner it
// stores its own body rows (and, for the preconditioner, its own periphery rows) into every window and meets its peers
// at the rows phase; from there on the complete x_bodies / x_shell are in its own window.  Body outputs land in the
// whole body layout (sys_rb) and are compacted to the own rows in one launch.  skb_mflow drives these calls on its
// members (skb_mflow.cu).

Group::Ranges skb::group_ranges(const skb_flow *fl) { return {fl->fa, fl->fb, fl->sa, fl->sb, fl->ba, fl->bb}; }

long long skb::group_local_size(const skb_flow *fl) {
    return 4 * (fl->fb - fl->fa) + 3 * (fl->sb - fl->sa) + fl->grp.body_rows();
}

// the refusals of the group matvec (stresslet_plus_complementary in dn) and preconditioner (M_inv in dn, the inverses),
// all before any launch; then the flow's device is current and its target ranges resolved
int skb::group_system_args(skb_flow *fl, skb_dense *dn, const char *who, bool precondition) {
    CUDA_TRY(cudaSetDevice(fl->dev));
    SKB_TRY(fl->grp.connected());
    SKB_TRY(prepare_matvec_targets(fl));
    if (!fl->grp.rows_for(group_ranges(fl)))
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_group_set_body_operators after skb_flow_group_init and after "
                                          "every change of the target ranges", who);
    SKB_TRY(system_ready(fl, who, kGroupCalls, precondition));
    return fl->sb > fl->sa ? dense_rows(fl, dn, who, precondition) : SKB_OK;
}

int skb::flow_gmres_size(skb_flow *fl, const char *who, long long *n, std::array<long long, 6> *key) {
    CUDA_TRY(cudaSetDevice(fl->dev));
    if (!fl->grp.member()) {
        *n = solution_size(fl);
        *key = {};
        return SKB_OK;
    }
    SKB_TRY(prepare_matvec_targets(fl));
    if (!fl->grp.rows_for(group_ranges(fl)))
        return set_error(SKB_ERR_INVALID, "%s: a group member's rows are laid out by skb_flow_group_set_body_operators "
                                          "(after skb_flow_group_init and every change of the target ranges)", who);
    *n = group_local_size(fl);
    *key = group_ranges(fl);
    return SKB_OK;
}

int skb::flow_member_lay_out_rows(skb_flow *fl, const char *who, const int *n_nodes, int n_bodies) {
    if (!fl->grp.member())
        return SKB_OK;
    CUDA_TRY(cudaSetDevice(fl->dev));
    OwnFibers own;
    SKB_TRY(own_fibers(fl, who, own)); // the target ranges resolved, the window's layout checked
    std::vector<RowPiece> pieces;
    if (!body_row_pieces(n_nodes, n_bodies, fl->ba, fl->bb, pieces))
        return set_error(SKB_ERR_STATE, "%s: the body rows [%lld, %lld) make %d pieces (at most %d)", who, fl->ba,
                         fl->bb, (int)pieces.size(), kMaxRowPieces);
    long long sol = 0;
    for (int b = 0; b < n_bodies; ++b)
        sol += 3LL * n_nodes[b] + 6;
    // every buffer of the local-vector calls at its final size now: none of them allocates while a peer on this device
    // may wait on a flag (the warm-up sized the matvec flow's own)
    SKB_TRY(fl->sys_rb.ensure((size_t)sol * 8 + 8));
    SKB_TRY(fl->tmp_b.ensure((size_t)(fl->bb - fl->ba) * 24 + 8)); // the matvec's own v_bodies rows
    SKB_TRY(fl->ft_sum.ensure((size_t)fl->n_bodies * 48 + 8));     // ... and its exchanged link forces
    SKB_TRY(load_dense_kernels()); // the preconditioner's M_inv rows (and the matvec's without the streamer)
    fl->grp.set_body_rows(pieces, group_ranges(fl));
    return SKB_OK;
}

extern "C" {

int skb_flow_group_set_body_operators(skb_flow *fl, const int *n_nodes, int n_bodies, const double *node_weights,
                                      const double *ex, const double *ey, const double *ez, const double *A_inv) {
    const char *who = "skb_flow_group_set_body_operators";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (!fl->grp.member())
        return skb_flow_set_body_operators(fl, n_nodes, n_bodies, node_weights, ex, ey, ez, A_inv);
    if (n_bodies != fl->n_bodies)
        return set_error(SKB_ERR_INVALID, "%s: %d bodies, skb_flow_set_bodies has %d", who, n_bodies, fl->n_bodies);
    if (n_bodies > 0 && (!n_nodes || !node_weights || !ex || !ey || !ez))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    CUDA_TRY(cudaSetDevice(fl->dev));
    OwnFibers own;
    SKB_TRY(own_fibers(fl, who, own)); // the target ranges resolved, the window's layout checked
    SKB_TRY(fl->bodies.set_operators(n_nodes, n_bodies, fl->n_body, fl->h_r_body.data(), fl->h_centers.data(),
                                     node_weights, ex, ey, ez, A_inv, fl->stream, fl->ba, fl->bb));
    SKB_TRY(flow_member_lay_out_rows(fl, who, n_nodes, n_bodies));
    SKB_TRY(rhs_buffers(fl)); // the RHS's buffers at their final size too
    return fl->ops.size_rhs(own.count());
}

int skb_flow_group_set_body_frames(skb_flow *fl, const int *n_nodes, int n_bodies, const double *node_pos_ref,
                                   const double *node_normal_ref, const double *node_weights, const double *ex0,
                                   const double *ey0, const double *ez0, const double *A_inv0) {
    const char *who = "skb_flow_group_set_body_frames";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (!fl->grp.member())
        return skb_flow_set_body_frames(fl, n_nodes, n_bodies, node_pos_ref, node_normal_ref, node_weights, ex0, ey0,
                                        ez0, A_inv0);
    CUDA_TRY(cudaSetDevice(fl->dev));
    OwnFibers own;
    SKB_TRY(own_fibers(fl, who, own)); // the target ranges resolved, the window's layout checked
    SKB_TRY(body_frames(fl, who, n_nodes, n_bodies, node_pos_ref, node_normal_ref, node_weights, ex0, ey0, ez0,
                        A_inv0));
    SKB_TRY(flow_member_lay_out_rows(fl, who, n_nodes, n_bodies));
    SKB_TRY(rhs_buffers(fl)); // as skb_flow_group_set_body_operators does
    return fl->ops.size_rhs(own.count());
}

int skb_flow_group_place_bodies(skb_flow *fl, const double *centers, const double *orientations) {
    const char *who = "skb_flow_group_place_bodies";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (!fl->grp.member())
        return skb_flow_place_bodies(fl, centers, orientations);
    std::vector<double> R;
    SKB_TRY(placement_args(fl, who, centers, orientations, R));
    SKB_TRY(place_bodies(fl, centers, orientations, R));
    return prepare_matvec_targets(fl); // the new body rows' targets now, not at the first matvec
}

int skb_flow_group_set_fiber_links(skb_flow *fl, const int *body, const double *site, const double *bending_rigidity) {
    const char *who = "skb_flow_group_set_fiber_links";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (!fl->grp.member())
        return skb_flow_set_fiber_links(fl, body, site, bending_rigidity);
    CUDA_TRY(cudaSetDevice(fl->dev));
    OwnFibers own;
    SKB_TRY(own_fibers(fl, who, own));
    if (body && own.count() > 0 && (!site || !bending_rigidity))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    return fl->bodies.set_links(own, fl->ops, fl->n_bodies, fl->h_centers.data(), body, site, bending_rigidity,
                                fl->stream);
}

int skb_flow_group_apply_system_matvec_device(skb_flow *fl, skb_dense *dn, const double *d_x_local, double eta,
                                              double *d_res_local, void *stream) {
    const char *who = "skb_flow_group_apply_system_matvec_device";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (!fl->grp.member())
        return skb_flow_apply_system_matvec_device(fl, dn, d_x_local, eta, d_res_local, stream);
    SKB_TRY(group_system_args(fl, dn, who, false));
    if (!(eta > 0))
        return set_error(SKB_ERR_INVALID, "%s: eta = %g", who, eta);
    if (group_local_size(fl) > 0 && (!d_x_local || !d_res_local))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    begin_stats(fl);
    return device_frame(fl, stream, [&]() -> int {
        Group &G = fl->grp;
        const long long n_fw = fl->fb - fl->fa, n_sw = fl->sb - fl->sa;
        const double *x_fib = d_x_local, *x_shell = x_fib + 4 * n_fw, *x_body = x_shell + 3 * n_sw;
        double *res_fib = d_res_local, *res_shell = res_fib + 4 * n_fw, *res_body = res_shell + 3 * n_sw;
        double *full = (double *)fl->sys_rb.ptr;
        const bool bodies = fl->n_bodies > 0;
        SKB_TRY(G.begin());
        if (bodies) { // the complete x_bodies in every window first: the links read the bodies' U, w before barrier A
            SKB_TRY(G.store_rows(x_body, nullptr, 0, 0, fl->fib[1].info.num_sms, fl->cur, &fl->launches));
            SKB_TRY(G.rows_barrier(true, true, fl->cur, &fl->launches));
        }
        fl->grp_open = true; // matvec_core's push, barriers and pull run in this epoch
        const int rc = member_system_matvec_core(fl, dn, x_fib, x_shell, bodies ? G.x_body() : nullptr, eta, res_fib,
                                                 res_shell, full);
        fl->grp_open = false;
        SKB_TRY(rc);
        return bodies ? G.compact_rows(full, res_body, fl->cur, &fl->launches) : SKB_OK;
    });
}

int skb_flow_group_apply_system_preconditioner_device(skb_flow *fl, skb_dense *dn, const double *d_x_local,
                                                      double *d_y_local, void *stream) {
    const char *who = "skb_flow_group_apply_system_preconditioner_device";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (!fl->grp.member())
        return skb_flow_apply_system_preconditioner_device(fl, dn, d_x_local, d_y_local, stream);
    SKB_TRY(group_system_args(fl, dn, who, true));
    if (group_local_size(fl) > 0 && (!d_x_local || !d_y_local))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    begin_stats(fl);
    return device_frame(fl, stream, [&]() -> int {
        Group &G = fl->grp;
        const long long n_fw = fl->fb - fl->fa, n_sw = fl->sb - fl->sa;
        const double *x_fib = d_x_local, *x_shell = x_fib + 4 * n_fw, *x_body = x_shell + 3 * n_sw;
        double *y_fib = d_y_local, *y_shell = y_fib + 4 * n_fw, *y_body = y_shell + 3 * n_sw;
        double *full = (double *)fl->sys_rb.ptr;
        // the complete x_shell and x_bodies in every window; the fibers' A_^-1 runs while the peers' rows arrive
        SKB_TRY(G.begin());
        SKB_TRY(G.store_rows(x_body, n_sw > 0 ? x_shell : nullptr, fl->sa, n_sw, fl->fib[1].info.num_sms,
                             fl->cur, &fl->launches));
        SKB_TRY(G.rows_barrier(true, false, fl->cur, &fl->launches));
        SKB_TRY(fl->ops.precondition(x_fib, y_fib, fl->cur, &fl->launches));
        SKB_TRY(G.rows_barrier(false, true, fl->cur, &fl->launches));
        if (n_sw > 0) { // the member's rows of M_inv times the complete x_shell
            SKB_TRY(skb_dense_apply_device(dn, SKB_DENSE_M_INV, G.x_shell(), nullptr, y_shell, fl->cur));
            fl->launches += 1;
        }
        if (fl->n_bodies > 0) {
            SKB_TRY(fl->bodies.precondition(G.x_body(), full, fl->cur, &fl->launches));
            SKB_TRY(G.compact_rows(full, y_body, fl->cur, &fl->launches));
        }
        return SKB_OK;
    });
}

int skb_flow_group_build_system_rhs_device(skb_flow *fl, const skb_fiber_params *params, const double *v_growth,
                                           const double *force_scale, const double *d_f_external,
                                           const double *d_body_forces, const double *d_body_torques, double dt,
                                           double eta, double *d_rhs_local, void *stream) {
    const char *who = "skb_flow_group_build_system_rhs_device";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    if (!fl->grp.member())
        return skb_flow_build_system_rhs_device(fl, params, v_growth, force_scale, d_f_external, d_body_forces,
                                                d_body_torques, dt, eta, d_rhs_local, stream);
    if (!(dt > 0) || !(eta > 0))
        return set_error(SKB_ERR_INVALID, "%s: dt = %g, eta = %g (both must be > 0)", who, dt, eta);
    CUDA_TRY(cudaSetDevice(fl->dev));
    SKB_TRY(fl->grp.connected());
    OwnFibers own;
    SKB_TRY(own_fibers(fl, who, own));
    if (!fl->grp.rows_for(group_ranges(fl)))
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_group_set_body_operators after skb_flow_group_init and after "
                                          "every change of the target ranges", who);
    if (fl->n_bodies > 0 && !fl->bodies.has_operators())
        return set_error(SKB_ERR_INVALID, "%s: call skb_flow_group_set_body_operators after skb_flow_set_bodies (the "
                                          "body rows are laid out by its node counts)", who);
    if ((own.count() > 0 && !params) || (group_local_size(fl) > 0 && !d_rhs_local))
        return set_error(SKB_ERR_INVALID, "%s: NULL argument", who);
    begin_stats(fl);
    return device_frame(fl, stream, [&]() -> int {
        const long long n_fw = fl->fb - fl->fa, n_sw = fl->sb - fl->sa;
        double *rhs_fib = d_rhs_local, *rhs_shell = rhs_fib + 4 * n_fw, *rhs_body = rhs_shell + 3 * n_sw;
        double *full = (double *)fl->sys_rb.ptr;
        // the fiber block's checks come first inside system_rhs_core, before its first launch; F_T complete, as they
        // are
        SKB_TRY(system_rhs_core(fl, own, params, v_growth, force_scale, own.count() > 0 ? d_f_external : nullptr,
                                fl->n_bodies ? d_body_forces : nullptr, fl->n_bodies ? d_body_torques : nullptr, dt,
                                eta, rhs_fib, rhs_shell, full));
        return fl->n_bodies > 0 ? fl->grp.compact_rows(full, rhs_body, fl->cur, &fl->launches) : SKB_OK;
    });
}

} // extern "C"


/*
 * skelly_b200_flow.h -- C ABI of the device-resident flow() layer: the three container flows that
 * System::apply_matvec evaluates every GMRES iteration, and their fused sum.
 *
 *   reference (SkellySim)                                                       here
 *   --------------------------------------------------------------------------  -----------------------
 *   FiberContainerFiniteDifference::flow   fiber_container_finite_difference.cpp:172-214   skb_flow_fibers
 *   Periphery::flow                        periphery.cpp:55-79                             skb_flow_periphery
 *   BodyContainer::flow (spherical/ellipsoidal)  body_container.cpp:269-411,471-477        skb_flow_bodies
 *   System::apply_matvec, hydrodynamic part      system.cpp:284-316                        skb_flow_matvec
 *
 * A skb_flow object holds the geometry of ONE timestep on the device (node positions, normals, quadrature
 * weights, body centres); positions only change in System::step (system.cpp:486-489), so every GMRES
 * iteration ships densities/forces only.  Layouts are the reference's: Eigen column-major 3 x n == AoS xyz.
 * Velocities returned here are the reference's flow() return values, i.e. they INCLUDE the 1/eta of the
 * evaluator wrappers (kernels.cpp:358,365).
 */
#ifndef SKELLY_B200_FLOW_H
#define SKELLY_B200_FLOW_H

#include "skelly_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct skb_flow skb_flow;

SKB_API int skb_flow_create(int device, skb_flow **out);
SKB_API int skb_flow_destroy(skb_flow *fl);

/* ---- geometry, once per timestep --------------------------------------------------------------------- */
/* r_fib: 3 x N_f node positions of all fibers, concatenated in container order; n_nodes[f] nodes and
 * length[f] per fiber (trapezoid weights 0.5 L weights_0 are formed on the device,
 * fiber_container_finite_difference.cpp:185-193).  n_fibers == 0 is allowed (flow returns zeros, :178-179). */
SKB_API int skb_flow_set_fibers(skb_flow *fl, const double *r_fib, const int *n_nodes, const double *length,
                                int n_fibers);
/* periphery quadrature nodes and (inward) normals, periphery.hpp node_pos_ / node_normal_ */
SKB_API int skb_flow_set_periphery(skb_flow *fl, const double *node_pos, const double *node_normal, int64_t n_nodes);
/* all body surface nodes / normals concatenated [spherical..., ellipsoidal...] (body_container.cpp:286-290),
 * and the body centres (get_local_center_positions) */
SKB_API int skb_flow_set_bodies(skb_flow *fl, const double *node_pos, const double *node_normal, int64_t n_nodes,
                                const double *centers, int n_bodies);

/* ---- the three flows at arbitrary targets (velocity_at_targets / listener path, system.cpp:330-384) ------
 * Targets are cached on the device and re-uploaded only when they differ from the previous call's (the same
 * full compare the reference's FMM functor does, kernels.hpp:81-83). */
SKB_API int skb_flow_fibers(skb_flow *fl, const double *r_trg, int64_t n_trg, const double *fib_forces, double eta,
                            int subtract_self, double *vel);
SKB_API int skb_flow_periphery(skb_flow *fl, const double *r_trg, int64_t n_trg, const double *density, double eta,
                               double *vel);
/* densities: 3 x N_b body-node densities; forces_torques: 6 x n_bodies (net force then torque per body,
 * body_container.cpp:128-135) */
SKB_API int skb_flow_bodies(skb_flow *fl, const double *r_trg, int64_t n_trg, const double *densities,
                            const double *forces_torques, double eta, double *vel);

/* System::velocity_at_targets (system.cpp:330-384), hydrodynamic part: fiber flow WITHOUT self-term subtraction +
 * body flow + periphery flow at arbitrary targets (system.cpp:355-359; point/background sources are analytic
 * add-ons outside this library).  This is what the listener and the streamline integrator evaluate.  Any class may
 * be empty; one upload of the strengths, one download of the velocities. */
SKB_API int skb_flow_velocity_at_targets(skb_flow *fl, const double *r_trg, int64_t n_trg, const double *fib_forces,
                                         const double *shell_density, const double *body_densities,
                                         const double *body_forces_torques, double eta, double *vel);

/* Optional analytic add-ons of velocity_at_targets (system.cpp:358-359) and of skb_flow_build_system_rhs: point
 * forces/torques (PointSourceContainer::flow, point_source.cpp:16-54: regularised Oseen contraction + rotlet; the caller
 * passes the points that are alive at the current time) and the linear background flow (BackgroundSource::flow,
 * background_source.cpp:15-24: u_j = uniform_j + r[components_j] * scale_factor_j).  n_points == 0 / NULL clears. */
SKB_API int skb_flow_set_point_sources(skb_flow *fl, const double *positions, const double *forces,
                                       const double *torques, int n_points);
SKB_API int skb_flow_set_background(skb_flow *fl, const int *components, const double *scale_factor,
                                    const double *uniform);

/* ---- the listener: velocity field, streamlines and vortex lines of one frame (listener.cpp:86-136) ----------------
 * A frame holds the strengths of one solution on the device.  fib_forces, shell_density, body_densities and
 * body_forces_torques are those of skb_flow_velocity_at_targets (f_on_fibers, the periphery's solution, the body
 * densities, the link-plus-external forces and torques); body_velocities is [U; omega] per body (6 x n_bodies, the tail
 * of the body rows of the solution).  body_kind[b] is 0 (no interior test), 1 (sphere: |dx| < body_radii[3b]) or
 * 2 (ellipsoid: sum dx_i^2 / r_i^2 < 1 on the world-frame dx, the body's orientation ignored as in system.cpp:362-381);
 * body_radii is 3 per body.  Point sources and the background flow of the flow at the time of the requests are part
 * of the velocity.  The frame goes stale (the requests refuse with SKB_ERR_STATE) when the geometry, the point sources
 * or the background flow change after it was set. */
SKB_API int skb_flow_set_listener_frame(skb_flow *fl, const double *fib_forces, const double *shell_density,
                                        const double *body_densities, const double *body_forces_torques,
                                        const double *body_velocities, const int32_t *body_kind,
                                        const double *body_radii, double eta);
/* The frame of the installed geometry and a step's solution, built on the device as the reference's listener unpacks a
 * trajectory frame (trajectory_reader.cpp:150-249) and System::velocity_at_targets forms its strengths (system.cpp:
 * 339-356):
 *   fib_forces    = fc.apply_fiber_force([x; y; z; T]) per fiber, with x, y, z the flow's installed positions and T
 *                   `tension` (N_f values, as skb_flow_step returns it) -- not the fiber block of the solution -- and
 *                   force_operator_ built at those positions by skb_flow_build_fiber_operators(params, dt, eta);
 *                   plus the fiber-periphery repulsion at the installed positions when periphery_interaction != 0
 *                   (needs skb_flow_set_periphery_shape); no motor force;
 *   body_forces_torques = the link forces and torques of calculate_link_conditions([x; y; z; T], x_bodies) at the
 *                   links of skb_flow_set_fiber_links -- and no external forces or torques, as the reference computes
 *                   calculate_external_forces_torques there and does not pass it to the body flow;
 *   shell_density = the shell block of x; body_densities = the first 3 n_b entries of each body's block of x;
 *   body_velocities = the last six entries of each body's block of x (SphericalBody::step's velocity_ and
 *                   angular_velocity_).
 * x is the whole solution vector as skb_flow_step returns it; only its shell and body blocks are read.  body_kind and
 * body_radii are those of skb_flow_set_listener_frame.  The frame is the one skb_flow_set_listener_frame would hold for
 * these strengths, with the same staleness and the same requests.  The call leaves A_, force_operator_ and xs_ of the
 * installed geometry resident, built without their inverse: skb_flow_apply_fiber_preconditioner and the system calls
 * that precondition refuse until the next skb_flow_build_fiber_operators (skb_flow_step builds its own).  It returns once the frame is complete; the _device form
 * takes d_tension and d_x on the flow's device, waits for `stream` first and never moves them through the host.
 * Refused (SKB_ERR_INVALID, before any launch): dt or eta not finite and > 0, a non-finite tension (host form), a bad
 * body_kind or body_radii, NULL inputs of a non-empty block, a group member or a target window or ranges, fibers without
 * their class derivatives or with bad params, bodies without operators, fibers and bodies without
 * skb_flow_set_fiber_links for the current geometry, periphery_interaction with fiber nodes but no periphery shape.
 * Any refusal or failure leaves no frame.  An empty block needs none of its set-up. */
struct skb_fiber_params; /* below, with skb_flow_build_fiber_operators */
SKB_API int skb_flow_set_listener_state(skb_flow *fl, const struct skb_fiber_params *params, double dt, double eta,
                                        const double *tension, const double *x, const int32_t *body_kind,
                                        const double *body_radii, int32_t periphery_interaction);
SKB_API int skb_flow_set_listener_state_device(skb_flow *fl, const struct skb_fiber_params *params, double dt,
                                               double eta,
                                               const double *d_tension, const double *d_x, const int32_t *body_kind,
                                               const double *body_radii, int32_t periphery_interaction, void *stream);
/* System::velocity_at_targets (system.cpp:330-384) on the frame: skb_flow_velocity_at_targets's velocity, and at a
 * target inside a body (bodies in the library's order, the last match wins) the body's rigid motion U + omega x dx. */
SKB_API int skb_flow_listener_velocity(skb_flow *fl, const double *r_trg, int64_t n_trg, double *vel);
/* The velocity gradient and the pressure of the listener's frame at n_trg targets (3 each):
 * grad[9 t + 3 i + j] = d u_i / d x_j, pressure[t].  Same frame, staleness and refusals as
 * skb_flow_listener_velocity; n_trg == 0 is a no-op.  The gradient is the analytic one of every source of that
 * velocity (fibers' Stokeslets, the bodies' and the periphery's stresslets, the bodies' net forces and torques, the
 * point sources' regularised Oseen and rotlet kernels, the background flow); the pressure is that of the Stokeslets,
 * stresslets and point forces, p -> 0 far from every source.  A coincident source adds exactly 0 to every output.  At a
 * target inside a body (the velocity's test and order) the gradient is the rigid motion's, eps_ikj omega_k, and the
 * pressure is NaN.  Both outputs are written for every target. */
SKB_API int skb_flow_listener_gradient(skb_flow *fl, const double *r_trg, int64_t n_trg, double *grad,
                                       double *pressure);

/* StreamLine::compute / VortexLine::compute (streamline.cpp) for n_lines seeds x0 (3 each) at once: odeint's
 * integrate_adaptive with the controlled Cash-Karp 5(4) stepper (default error checker and step adjuster, 500 failed
 * tries end a line), from t = 0 to +t_final and, with back_integrate, to -t_final.  kind 0 integrates the velocity,
 * kind 1 the vorticity (central differences at +-1e-7, streamline.cpp:16-35); the integration stops where
 * |velocity| > 1e3.  Output per line i, left-aligned in rows of 2 max_points - 1 points: the back points reversed
 * without their copy of x0, then the forward points (join_back_and_forward); x and val are 3 per point (val: the
 * velocity or the vorticity there), t 1 per point; n_points[i] points.  status[2 i + d] (d = 0 back, 1 forward): 0
 * reached +-t_final, 1 |velocity| > 1e3, 2 500 failed tries, 3 max_points points in that direction (this library's
 * cap: the reference has none); the back status is 0 without back_integrate. */
typedef struct {
    double dt_init, t_final, abs_err, rel_err;
    int32_t back_integrate, max_points;
} skb_line_request;
enum { SKB_STREAMLINE = 0, SKB_VORTEXLINE = 1 };
SKB_API int skb_flow_listener_lines(skb_flow *fl, int kind, const double *x0, int32_t n_lines,
                                    const skb_line_request *req, double *x, double *t, double *val, int32_t *n_points,
                                    int32_t *status);

/* ---- fused matvec flow -------------------------------------------------------------------------------
 * v_all over targets [fibers | periphery | bodies] (get_node_maps, system.cpp:234-241):
 *   v_all  = fiber flow (all targets, self term subtracted)
 *   v_fib, v_body += periphery flow   (shell sources never act on shell targets, system.cpp:301-315)
 *   v_all += body flow
 * Any class may be empty.  One H2D of the four strength arrays, one D2H of v_all; everything in between stays
 * on the device. */
SKB_API int skb_flow_matvec(skb_flow *fl, const double *fib_forces, const double *shell_density,
                            const double *body_densities, const double *body_forces_torques, double eta,
                            double *v_all);

/* The (fiber node, periphery node) pairs of a matvec are visited twice -- the fibers' Stokeslets act on the periphery
 * (system.cpp:299) and the periphery's stresslets on the fibers (system.cpp:304,313-315).  By default (mode -1: when both
 * classes are large enough and all fiber rows are in the target list) one kernel evaluates both directions from one pass
 * over the pairs (37 instead of 49 FP64 instructions per visited pair); results agree with the two separate evaluator
 * calls to rounding.  0: never (two calls, as the reference issues them); 1: whenever applicable. */
SKB_API int skb_flow_set_cross(skb_flow *fl, int mode);

/* Opt-in (SURVEY.md 8f N3): the matvec's fiber self term.  fused == 0 (default): the reference's way -- all pairs,
 * then `vel -= fib.stokeslet_ * wf` per fiber (fiber_container_finite_difference.cpp:203-210) on the device.
 * fused != 0: the pair kernels skip every intra-fiber pair (per-node fiber id compared in the integer pipe), nothing is
 * subtracted: no cancellation of the O(1/ds) near-neighbour terms, and N_f * n fewer pairs.  The two agree except where
 * the reference's regularised branch acts (distinct nodes of one fiber closer than 1e-5, kernels.cpp:176-184).  Applies
 * to skb_flow_matvec / skb_flow_apply_matvec with all fiber nodes in the target list. */
SKB_API int skb_flow_set_self_exclusion(skb_flow *fl, int fused);
/* Overlap of the HBM-bound dense operator with the FP64-bound pair kernels (default on): skb_flow_apply_matvec_dense /
 * _device hand stresslet_plus_complementary * x_shell (Periphery::matvec, periphery.cpp:38-47) to the background row
 * streamer (skb_dense_apply_background_device) on a side stream as soon as x_shell is complete on the device, and add
 * v_shell when both are there.  0: one GEMV kernel at the end of the stream instead (the round-1 order).  The results
 * differ in the last bits only (another summation order inside a row). */
SKB_API int skb_flow_set_overlap(skb_flow *fl, int on);

/* Restrict the matvec to rows [begin, end) of the target list [fibers | periphery | bodies] (end < 0: all).
 * For one-rank-per-GPU hosts: every rank loads the full geometry, all-gathers the strengths, and evaluates its own
 * block of targets; v_all / d_v_window then has (end - begin) rows.  The self-term subtraction is applied to the
 * fiber rows inside the window. */
SKB_API int skb_flow_set_target_window(skb_flow *fl, int64_t begin, int64_t end);

/* The reference's own MPI decomposition as three ranges (whole fibers [fiber_begin, fiber_end) of the container,
 * fiber_container_finite_difference.cpp:102-120; periphery rows, periphery.cpp:387-400; body-node rows -- all on
 * rank 0 in the reference): the target list of this flow becomes [own fiber nodes | own shell rows | own body rows]
 * and v_all / d_v_window has that many rows in that order.  Replaces a window set earlier (and vice versa). */
SKB_API int skb_flow_set_target_ranges(skb_flow *fl, int fiber_begin, int fiber_end, int64_t shell_begin,
                                       int64_t shell_end, int64_t body_begin, int64_t body_end);

/* Device-pointer form of skb_flow_matvec: all inputs and the output already on this flow's device; asynchronous on
 * `stream` (cudaStream_t as void*, used verbatim).  d_body_forces / d_body_torques are 3 x n_bodies each. */
SKB_API int skb_flow_matvec_device(skb_flow *fl, const double *d_fib_forces, const double *d_shell_density,
                                   const double *d_body_densities, const double *d_body_forces,
                                   const double *d_body_torques, double eta, double *d_v_window, void *stream);

/* ---- multi-GPU groups: one skb_flow per GPU, exchange through peer memory (NVLink / NVSwitch) -----------------
 * Every member holds the full geometry (skb_flow_set_fibers / _periphery / _bodies with identical arguments) and owns
 * whole fibers, periphery rows and body rows (skb_flow_set_target_ranges).  Per matvec each member packs the strengths
 * of ITS fibers / periphery rows once and stores them straight into all members' windows (pack + all-gather in one
 * kernel), evaluates its block rows of the symmetric fiber-fiber interaction and its own remainder rows from local
 * memory, and finally adds up the partial velocities of its own fiber rows from all windows (reduce-scatter fused
 * with the accumulation).  No library collective is on the path; ordering is by epoch flags in the windows.
 *   same process (what the reference's one-rank rule for direct evaluators admits, system.cpp:618-623): create one
 *     flow per device, skb_flow_group_init on each, then skb_flow_group_connect every ordered pair -- or simply use
 *     skb_mflow_* below, which does all of that;
 *   one process per GPU: skb_flow_group_init, skb_flow_group_export -> exchange the 64-byte handles by any means
 *     (MPI_Allgather, torch.distributed) -> skb_flow_group_import for every peer.
 * skb_flow_group_init must follow the geometry calls (the window is laid out for their fiber and periphery node counts
 * and for the number of bodies, whose link forces it carries; positions may change later, counts may not: a member
 * whose counts changed refuses its matvec until the group is initialised again -- skb_mflow does that itself, and then
 * wants its fiber operators set again).  In a group, the *_device entry points take the OWN slices: fiber forces / x_fibers of
 * the own fibers, periphery density of the own rows; body inputs are complete on every member.  All members must issue
 * the same sequence of matvec calls (like any collective). */
#define SKB_FLOW_IPC_HANDLE_BYTES 64
SKB_API int skb_flow_group_init(skb_flow *fl, int rank, int size);
SKB_API int skb_flow_group_export(skb_flow *fl, void *handle_64_bytes);
SKB_API int skb_flow_group_import(skb_flow *fl, int peer_rank, const void *handle_64_bytes);
SKB_API int skb_flow_group_connect(skb_flow *fl, int peer_rank, skb_flow *peer);
/* one matvec of this member alone (no flags, zero strengths) so that every buffer reaches its final size before the
 * first real matvec: device-wide synchronisation by cudaMalloc / cudaFree must not happen while a peer ON THE SAME
 * DEVICE waits on a flag.  Call after the ranges are set and all peers are connected; skb_mflow does it itself. */
SKB_API int skb_flow_group_warmup(skb_flow *fl);
/* profiling aid: from now on evaluate this member's share alone (no flags, own window only): the per-rank device time
 * of an n-way group measured on ONE GPU.  The results are the member's partial view, not the group's. */
SKB_API int skb_flow_group_set_solo(skb_flow *fl, int solo);
/* after synchronising: *missing_peer = rank of a member whose flag never arrived within the time-out (a flag wait
 * gives up after ~10 s instead of hanging the GPU), or -1 */
SKB_API int skb_flow_group_error(skb_flow *fl, int *missing_peer);

/* ---- per-fiber dense operators on the device (SURVEY.md §8f N2) ------------------------------------------
 * The O(N_f n^2) host work of one GMRES iteration -- FiberContainerFiniteDifference::apply_fiber_force
 * (fiber_container_finite_difference.cpp:272-287) and ::matvec (:216-232 -> FiberFiniteDifference::matvec,
 * fiber_finite_difference.cpp:276-312) -- as batched GEMVs over operators that stay resident for the timestep.
 * All matrices are COLUMN-MAJOR, exactly as Eigen stores the reference's members, so `.data()` goes in as is.
 *
 * skb_flow_set_fiber_class: the per-node-count constants FiberFiniteDifference::matrices_.at(n)
 *   (fiber_finite_difference.cpp:537-555): D_1_0 (n x n) and P_downsample_bc ((4n-14) x 4n).  Call once per
 *   distinct n (n >= 4), any time before skb_flow_set_fiber_operators.  The matrices are uploaded at once,
 *   after the work in flight on the flow's device has finished (the fiber kernels may still read the previous ones),
 *   so the call can also return SKB_ERR_CUDA.
 * skb_flow_set_fiber_operators: once per timestep, after skb_flow_set_fibers (which defines the fibers and their
 *   node counts): A = concatenated A_ (4n x 4n each), force_operator = concatenated force_operator_ (3n x 4n
 *   each), xs = 3 x N_f tangents xs_, length_prev[f] = length_prev_, plus_bc_velocity[f] = (bc_plus_.first ==
 *   Velocity). */
SKB_API int skb_flow_set_fiber_class(skb_flow *fl, int n_nodes, const double *D_1_0, const double *P_downsample_bc);
SKB_API int skb_flow_set_fiber_operators(skb_flow *fl, const double *A, const double *force_operator,
                                         const double *xs, const double *length_prev, const int *plus_bc_velocity);
/* fw (3 x N_f) = apply_fiber_force(x_fibers); x_fibers = per fiber [x; y; z; T] of 4n (fcfd.cpp:272-287) */
SKB_API int skb_flow_apply_fiber_force(skb_flow *fl, const double *x_fibers, double *fw);
/* res (4 N_f) = fc.matvec(x_fibers, v_fibers, v_fib_boundary); v_fibers 3 x N_f, v_fib_boundary 7 x n_fibers
 * (fiber_link_conditions of BodyContainer::calculate_link_conditions) or NULL for none (fcfd.cpp:216-232) */
SKB_API int skb_flow_fiber_matvec(skb_flow *fl, const double *x_fibers, const double *v_fibers,
                                  const double *v_fib_boundary, double *res);
/* One rank per GPU: under skb_flow_set_target_ranges (or a window that cuts no fiber) the resident operators are those
 * of the rank's OWN fibers -- skb_flow_set_fiber_operators, skb_flow_apply_fiber_force and skb_flow_fiber_matvec then
 * take / return the arrays of the own fibers only (x: 4 per own node, fw / v: 3 per own node, link conditions: 7 per
 * own fiber), as the reference's local solution vectors do.  Device-pointer forms, asynchronous on `stream`:
 *   d_fw_own = apply_fiber_force(d_x_own)  ->  [caller all-gathers fw]  ->  skb_flow_matvec_device  ->
 *   d_res_own = fc.matvec(d_x_own, first own-fiber rows of d_v_window, d_link_own) */
SKB_API int skb_flow_apply_fiber_force_device(skb_flow *fl, const double *d_x_fibers, double *d_fw, void *stream);
SKB_API int skb_flow_fiber_matvec_device(skb_flow *fl, const double *d_x_fibers, const double *d_v_fibers,
                                         const double *d_v_fib_boundary, double *d_res, void *stream);

/* The fiber block of System::apply_preconditioner (system.cpp:248-262): FiberContainerFiniteDifference::
 * apply_preconditioner (fcfd.cpp:331-339) is `A_LU_.solve(x)` per fiber; here the solve is a GEMV over the explicit
 * inverse, `fib.A_LU_.inverse()` (column-major 4n x 4n per fiber, concatenated in the order of
 * skb_flow_set_fiber_operators), uploaded once per timestep.  As a preconditioner it is a fixed linear operator, so
 * GMRES is indifferent to the rounding difference between LU substitution and the inverse.  (The shell block is
 * skb_dense_apply(SKB_DENSE_M_INV); bodies stay on the host.) */
SKB_API int skb_flow_set_fiber_preconditioner(skb_flow *fl, const double *A_inv);
SKB_API int skb_flow_apply_fiber_preconditioner(skb_flow *fl, const double *x_fibers, double *y);
SKB_API int skb_flow_apply_fiber_preconditioner_device(skb_flow *fl, const double *d_x_fibers, double *d_y,
                                                       void *stream);

/* ---- the per-fiber operators built on the device ------------------------------------------------------------
 * What FiberContainerFiniteDifference::update_cache_variables and ::apply_bc_rectangular (fcfd.cpp:147-157,
 * 261-269) do per fiber on the host before every solve -- update_derivatives (fiber_finite_difference.cpp:62-68),
 * update_linear_operator (:97-187), update_force_operator (:317-335), the operator half of apply_bc_rectangular
 * (`A_ = P_downsample_bc * A_` plus the 14 boundary rows, :347-512) and update_preconditioner (`A_LU_.compute(A_)`,
 * :340) -- from the positions and lengths of the last skb_flow_set_fibers and a few scalars per fiber, instead of
 * uploading A_, force_operator_ and A_^-1 (about 1 GB per timestep at 3000 fibers x 32 nodes).  The fiber block of the
 * RHS (update_RHS and the RHS half of apply_bc_rectangular) is formed on the device too: skb_flow_build_fiber_rhs.
 *
 * skb_flow_set_fiber_class_derivatives: the higher derivative matrices of FiberFiniteDifference::matrices_.at(n)
 *   (:537-540), stored pre-transposed exactly like the reference (column-major n x n each).  The build needs them,
 *   and skb_flow_set_fiber_class, for every node count in use.  Uploaded like skb_flow_set_fiber_class's matrices;
 *   the operators stay. */
SKB_API int skb_flow_set_fiber_class_derivatives(skb_flow *fl, int n_nodes, const double *D_2_0,
                                                 const double *D_3_0, const double *D_4_0);

typedef struct skb_fiber_params {   /* one per fiber, 48 bytes */
    double length_prev;             /* length_prev_  (derivatives and fc.matvec)              */
    double bending_rigidity;        /* bending_rigidity_                                      */
    double radius;                  /* radius_ -> epsilon_ = radius_/length_ (hpp:140-144)    */
    double penalty_param;           /* penalty_param_                                         */
    double beta_tstep;              /* beta_tstep_                                            */
    int32_t minus_clamped;          /* bc_minus_ = (Velocity, AngularVelocity), else (Force, Torque) */
    int32_t plus_hinged;            /* bc_plus_  = (Velocity, Torque),          else (Force, Torque) */
} skb_fiber_params;

/* update_derivatives + update_linear_operator + update_force_operator + the operator part of apply_bc_rectangular +
 * update_preconditioner, for every fiber of this flow, on the device, from the positions and lengths of the last
 * skb_flow_set_fibers.  Leaves exactly the state skb_flow_set_fiber_operators followed by
 * skb_flow_set_fiber_preconditioner leaves (A_, force_operator_, xs_, length_prev, plus flag, A_^-1); either call
 * replaces what the other left.  Under skb_flow_set_target_ranges (or a window that cuts no fiber) it builds the own
 * fibers only and `params` holds the own fibers.  Refused (SKB_ERR_INVALID, before any launch): a node count without
 * skb_flow_set_fiber_class or skb_flow_set_fiber_class_derivatives, n < 8 (the D_4 stencil has 8 points) or n > 128,
 * a flag outside {0, 1}, a non-positive length_prev, radius, dt or eta.
 * The inverse is Gauss-Jordan elimination with partial pivoting (Eigen's PartialPivLU does not detect a singular A_
 * either, and neither does this): a STRAIGHT fiber that is both clamped at the minus end and hinged at the plus end has
 * a singular A_ (condition number ~1e18 for every n), and its inverse is meaningless.
 * skb_flow_last_stats afterwards: device_ms = the build's kernels, total_ms = with the upload of its per-fiber tables. */
SKB_API int skb_flow_build_fiber_operators(skb_flow *fl, const skb_fiber_params *params, double dt, double eta);

/* The fiber block of System::get_rhs (fcfd.cpp:319-328) as System::prep_state_for_solver leaves it (system.cpp:416-453):
 * RHS_ of every fiber after fc.update_rhs(dt, v_on_fibers, motor + f_external) and fc.apply_bcs(dt, v_on_fibers,
 * f_external) -- update_derivatives, FiberFiniteDifference::update_RHS (fiber_finite_difference.cpp:198-274) and the RHS
 * half of apply_bc_rectangular (:358-504) -- from the positions and lengths of the last skb_flow_set_fibers.
 *   rhs: 4 per own node, [x; y; z; T] per fiber in container order.  Rows [0, 4n-14) of a fiber are
 *        P_downsample_bc * RHS_ of update_RHS, rows [4n-14, 4n) the 14 boundary entries of the branches the flags of
 *        `params` select (the same flags as skb_flow_build_fiber_operators).
 *   params: as for skb_flow_build_fiber_operators (length_prev for xs_ / xss_, radius -> c_0 with length_).
 *   v_growth: v_growth_ per own fiber (s_dot = (1 + alpha) v_growth / 2); NULL: all zero.
 *   force_scale: force_scale_ per own fiber: the motor force force_scale_ xs_ (generate_constant_force,
 *        fcfd.cpp:160-169) is added to f_external in update_RHS only; NULL: no motors.
 *   v_on_fibers, f_external: 3 x N_own, the flow at the fiber nodes and the external force; NULL: the reference's empty
 *        matrix (`flow.size() == 0`).  The boundary entries see f_external alone.
 * Needs skb_flow_set_fiber_class and skb_flow_set_fiber_class_derivatives for every node count in use, not the
 * operators: it works whether they were uploaded, built or never set, and leaves them and their inverse untouched.
 * Under skb_flow_set_target_ranges (or a window that cuts no fiber) every array holds the own fibers only.  Refused
 * (SKB_ERR_INVALID, before any launch): what skb_flow_build_fiber_operators refuses, a non-finite v_growth or
 * force_scale, NULL params or rhs.  skb_flow_last_stats afterwards: device_ms = the kernel, total_ms = with the uploads
 * of the inputs and the per-fiber tables and the download of rhs.
 * The _device form takes d_v_on_fibers, d_f_external and d_rhs on this flow's device and works on `stream`.  Its small
 * per-fiber tables come from host memory: it returns once they are staged, without waiting for the kernel (not
 * capturable into a CUDA graph).  Its stats count the launch, with no timings. */
SKB_API int skb_flow_build_fiber_rhs(skb_flow *fl, const skb_fiber_params *params, const double *v_growth,
                                     const double *force_scale, const double *v_on_fibers, const double *f_external,
                                     double dt, double eta, double *rhs);
SKB_API int skb_flow_build_fiber_rhs_device(skb_flow *fl, const skb_fiber_params *params, const double *v_growth,
                                            const double *force_scale, const double *d_v_on_fibers,
                                            const double *d_f_external, double dt, double eta, double *d_rhs,
                                            void *stream);

/* read the resident operators back, same layouts as skb_flow_set_fiber_operators / _preconditioner (own fibers);
 * NULL skips an array */
SKB_API int skb_flow_get_fiber_operators(skb_flow *fl, double *A, double *force_operator, double *xs, double *A_inv);

/* System::apply_matvec (system.cpp:269-324) with the fiber operators on the device:
 *   fw = apply_fiber_force(x_fibers); v_all = the fused flow of skb_flow_matvec;
 *   res_fibers = fc.matvec(x_fibers, v_fibers, fiber_link_conditions)
 * and the periphery / body rows of v_all returned for shell.matvec / bc.matvec (periphery.cpp:38-47 ->
 * skb_dense_apply; body_container.cpp matvec stays host glue).  Needs the full target window.  One H2D of the
 * solution-sized inputs, one D2H of the solution-sized outputs; fw and v_fibers never leave the device. */
SKB_API int skb_flow_apply_matvec(skb_flow *fl, const double *x_fibers, const double *shell_density,
                                  const double *body_densities, const double *body_forces_torques,
                                  const double *fiber_link_conditions, double eta, double *res_fibers,
                                  double *v_shell, double *v_bodies);

/* The same with Periphery::matvec on the device as well (skelly_b200_dense.h, single-device handle holding
 * SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY of size 3 N_s): returns res_shell = stresslet_plus_complementary_ * x_shell +
 * v_shell (system.cpp:319, periphery.cpp:38-47) instead of v_shell; x_shell and v_shell never leave the device. */
struct skb_dense;
SKB_API int skb_flow_apply_matvec_dense(skb_flow *fl, struct skb_dense *dn, const double *x_fibers,
                                        const double *x_shell, const double *body_densities,
                                        const double *body_forces_torques, const double *fiber_link_conditions,
                                        double eta, double *res_fibers, double *res_shell, double *v_bodies);

/* Device-pointer form of skb_flow_apply_matvec(_dense): everything already on this flow's device, asynchronous on
 * `stream`.  dn == NULL: d_out_shell = v_shell; else res_shell (the handle holds the own periphery rows x all columns).
 * Works for a whole system and for a group member (OWN slices: d_x_fibers / d_res_fibers 4 per own fiber node,
 * d_x_shell / d_out_shell 3 per own periphery row, d_fiber_link_conditions 7 per own fiber or NULL, d_v_bodies 3 per own
 * body row; body densities / forces / torques complete).  This is one GMRES iteration's operator apply with nothing
 * crossing PCIe (a12: solver_hydro.cpp:42-48 calls exactly this per iteration). */
SKB_API int skb_flow_apply_matvec_device(skb_flow *fl, struct skb_dense *dn, const double *d_x_fibers,
                                         const double *d_x_shell, const double *d_body_densities,
                                         const double *d_body_forces, const double *d_body_torques,
                                         const double *d_fiber_link_conditions, double eta, double *d_res_fibers,
                                         double *d_out_shell, double *d_v_bodies, void *stream);

/* ---- the whole solution vector: the body block and the fiber-body links on the device ------------------------
 * System::apply_matvec (system.cpp:269-324) and System::apply_preconditioner (system.cpp:248-262) on the reference's
 * whole solution vector [fibers | shell | bodies] (get_solution_maps, system.cpp:69-92): x_fibers 4 per fiber node
 * ([x; y; z; T] per fiber), x_shell 3 per periphery node, x_bodies (3 n_b + 6) per body ([densities (3 x n_b) ; U ;
 * omega], body_spherical.cpp:42-43).  What a caller computed on the host per GMRES iteration before --
 * BodyContainer::calculate_link_conditions (body_container.cpp:171-267), ::matvec (:487-504 -> body_spherical.cpp:39-63)
 * and ::apply_preconditioner (:510-521) -- runs on the device: this is A_fiber_hydro::apply / P_inv_hydro::apply
 * (solver_hydro.cpp:23-48) on a whole vector.  Spherical and ellipsoidal bodies have the same matvec and
 * preconditioner (body_ellipsoidal.cpp:37-63), so no body type is passed; deformable bodies do not exist here (the
 * reference throws for them, body_container.cpp:453).  K_ is never uploaded: K U = u + omega x (x_i - c) and
 * K^T lambda = [sum lambda_i ; sum (x_i - c) x lambda_i] follow from the node positions and centres of
 * skb_flow_set_bodies (body_spherical.cpp:74-86).
 *
 * Bodies are in ONE order, that of skb_flow_set_bodies, which must be the order of the bodies in the solution vector
 * (the reference's flow orders them spherical..., ellipsoidal..., body_container.cpp:278-290, the solution vector and
 * the link forces by `bodies`, :532-546; a caller with both kinds passes them to skb_flow_set_bodies in `bodies`
 * order).  Each bound fiber reads its own slice of x_fibers and writes its own column of the link conditions: the
 * reference's loop skips `i_fib++` and `xt_offset += 4 n` for a free fiber (:202-204, 262-263), which agrees with this
 * whenever the bound fibers precede the free ones.
 *
 * skb_flow_set_body_operators: once per timestep, after skb_flow_set_bodies (which drops them).  n_nodes[b] per body
 *   (summing to the node count of skb_flow_set_bodies, same order), node_weights (N_b, node_weights_), ex / ey / ez
 *   (3 x N_b each, AoS like the positions: ex_, ey_, ez_ of update_singularity_subtraction_vecs, body_spherical.cpp:
 *   168-181), A_inv: per body the column-major (3 n_b + 6)^2 inverse of A_ (update_preconditioner, :104-126),
 *   concatenated, or NULL (then the system preconditioner refuses bodies).  Refused: node counts that do not sum to
 *   skb_flow_set_bodies' count, a node weight <= 0, n_bodies other than skb_flow_set_bodies', a body too large for the
 *   preconditioner's GEMV (3 n_b + 6 > ~25000).
 * skb_flow_set_fiber_links: once per timestep, after skb_flow_set_fibers / _bodies / _fiber_class (each drops the links).
 *   Per fiber of the flow: body[f] (binding_site_.first, -1 = free), site (3 x n_fibers, the lab-frame nucleation site
 *   get_nucleation_site, unused for a free fiber), bending_rigidity[f] (bending_rigidity_; the table carries its own, so
 *   the links work whether the fiber operators were uploaded or built).  body == NULL: no fiber is bound.  Refused: a
 *   body index outside [-1, n_bodies), a bound fiber whose node count lacks skb_flow_set_fiber_class_derivatives (the
 *   link needs D_2_0 and D_3_0), a nucleation site at the body centre (site_pos.normalized(), :256, would divide by 0).
 *   xs_.col(0) comes from the resident fiber operators and length_ from skb_flow_set_fibers at every apply.
 *
 * skb_flow_apply_system_matvec(_device): res = A x, both of size 4 N_f + 3 N_s + sum(3 n_b + 6); dn holds
 *   SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY (3 N_s x 3 N_s, on the flow's device; may be NULL only if N_s == 0).
 * skb_flow_apply_system_preconditioner(_device): y = P^-1 x -- the fibers' A_^-1 (skb_flow_set_fiber_preconditioner or
 *   the build), the periphery's M_inv (dn holds SKB_DENSE_M_INV), the bodies' A_^-1 (a GEMV over the explicit inverse,
 *   like the fibers').
 * The host forms ship x once and res / y once; the _device forms are asynchronous on `stream`.  All four refuse
 * (SKB_ERR_INVALID, before any launch, earlier state untouched): a group member or a flow whose target window / ranges
 * do not cover every row (over several devices use skb_mflow_set_body_operators and its siblings below, or on one process
 * per GPU the skb_flow_group_* calls above), fiber operators not resident (with their inverse for the preconditioner), bodies without
 * skb_flow_set_body_operators, fibers and bodies without skb_flow_set_fiber_links (matvec), no A_inv (preconditioner),
 * dn == NULL or of the wrong shape with periphery nodes present.  The results are bitwise reproducible run to run: the
 * bodies' link forces are added per body in container order, without atomics.
 * An empty block needs none of its set-up, here, in skb_flow_build_system_rhs, in the skb_mflow_* system calls and in
 * the partial operator (skb_flow_apply_matvec(_device), skb_mflow_apply_matvec):
 * without fibers no fiber class, operators, preconditioner or links (a flow whose fibers all went away needs no new
 * upload: skb_flow_set_fibers drops the old operators); without periphery no dense handle (dn may be NULL); without
 * bodies no skb_flow_set_body_operators.  A group member (skb_flow_group_*) still calls
 * skb_flow_group_set_body_operators, which lays out its rows, and uploads the operators of its own fibers, none or
 * not.  The empty upload of an empty block is accepted and changes no result.  A solution vector of length 0 makes
 * every call return SKB_OK without a launch; its vectors may be NULL. */
SKB_API int skb_flow_set_body_operators(skb_flow *fl, const int *n_nodes, int n_bodies, const double *node_weights,
                                        const double *ex, const double *ey, const double *ez, const double *A_inv);
SKB_API int skb_flow_set_fiber_links(skb_flow *fl, const int *body, const double *site, const double *bending_rigidity);

/* ---- rigid bodies placed on the device (DESIGN.md §3.6) ---------------------------------------------------------
 * A rigid body's operators only move with it: placed at centre c and rotation R (x_i = c + R r_i, n_i = R n_i,ref,
 * body_spherical.cpp:146-159), its A_ is Q A_0 Q^T with Q = blockdiag(R, ..., R) (one R per node and two for [U; w]),
 * so A_^-1 = Q A_0^-1 Q^T, and per node E_i = [ex_i ey_i ez_i] = R E_i,0 R^T -- for spherical and ellipsoidal bodies
 * alike.  The flow keeps the body-frame operators resident and forms the placed ones from them on the device, always
 * from the body frame (never from the previous placement, so no rounding accumulates over the steps).
 *   skb_flow_set_body_frames: once per run, after skb_flow_set_bodies (n_bodies and the node total must be its).  Per
 *     body n_nodes[b]; per node the body-frame position node_pos_ref (node_positions_ref_, relative to the centre),
 *     normal node_normal_ref (node_normals_ref_) and node_weights (node_weights_), 3 / 3 / 1 per node; ex0 / ey0 / ez0
 *     and A_inv0 as skb_flow_set_body_operators takes them, of each body placed at identity orientation (any centre):
 *     place(anything, identity) then update_cache_variables.  A_inv0 may be NULL (then the system preconditioner
 *     refuses bodies).  Drops the resident body operators and links; keeps the body-frame E and inverses next to the
 *     placed ones (twice the inverses' memory).  Refused as skb_flow_set_body_operators.
 *   skb_flow_place_bodies: once per timestep.  centers 3 per body, orientations 4 per body, the unit quaternion
 *     (w, x, y, z) of orientation_.  R is Eigen's toRotationMatrix formula of it, the same R for the nodes and the
 *     operators.  Leaves the flow exactly as skb_flow_set_bodies(c + R r_ref, R n_ref, centers) followed by
 *     skb_flow_set_body_operators with the placed operators would: the fiber links are dropped (set them again with
 *     the new nucleation sites).  Refused (SKB_ERR_INVALID, before any launch, earlier state untouched): no frames, a
 *     body count or node total of skb_flow_set_bodies other than the frames', an orientation that is not finite or
 *     not unit within SKB_UNIT_QUATERNION_TOL (| w^2 + x^2 + y^2 + z^2 - 1 | above it: not a rotation), a group member
 *     (skb_flow_group_place_bodies).
 *   skb_flow_get_body_operators: the resident ex_ / ey_ / ez_ (3 x N_b each) and the resident inverses (concatenated,
 *     column-major; a group member's: those of the bodies it owns rows of), as skb_flow_set_body_operators took them.
 *     NULL skips an array.  Refused without resident operators (A_inv: without an inverse). */
#define SKB_UNIT_QUATERNION_TOL 1e-12
SKB_API int skb_flow_set_body_frames(skb_flow *fl, const int *n_nodes, int n_bodies, const double *node_pos_ref,
                                     const double *node_normal_ref, const double *node_weights, const double *ex0,
                                     const double *ey0, const double *ez0, const double *A_inv0);
SKB_API int skb_flow_place_bodies(skb_flow *fl, const double *centers, const double *orientations);
SKB_API int skb_flow_get_body_operators(skb_flow *fl, double *ex, double *ey, double *ez, double *A_inv);
SKB_API int skb_flow_apply_system_matvec(skb_flow *fl, struct skb_dense *dn, const double *x, double eta, double *res);
SKB_API int skb_flow_apply_system_matvec_device(skb_flow *fl, struct skb_dense *dn, const double *d_x, double eta,
                                                double *d_res, void *stream);
SKB_API int skb_flow_apply_system_preconditioner(skb_flow *fl, struct skb_dense *dn, const double *x, double *y);
SKB_API int skb_flow_apply_system_preconditioner_device(skb_flow *fl, struct skb_dense *dn, const double *d_x,
                                                        double *d_y, void *stream);

/* ---- the right-hand side of the whole system --------------------------------------------------------------------
 * System::prep_state_for_solver's RHS (system.cpp:398-458) as Solver::set_RHS lays it out (solver_hydro.cpp:51-61):
 * rhs has 4 N_f + 3 N_s + sum(3 n_b + 6) entries, the layout of the system calls above.  In the reference's order:
 *   v_all  = fc.flow(r_all, f_external, eta), the fiber self term subtracted (system.cpp:425; motor forces are not in
 *            this flow), + bc.flow(r_all, 0, F_T, eta): the bodies' centre Stokeslets and rotlets (:431-443)
 *   v_all += the point sources and the background flow of skb_flow_set_point_sources / _set_background (:445-446)
 *   fibers: skb_flow_build_fiber_rhs on the fiber rows of v_all (update_rhs with motor + f_external, apply_bcs with
 *           f_external, :451-453); shell: -v_shell (periphery.cpp:86); body b: [-v of its nodes ; 0 0 0 0 0 0]
 *           (body_spherical.cpp:134-138).  The periphery's densities and the link conditions do not enter.
 * The flow is skb_flow_matvec's (f_external, zero periphery and body densities, F_T): its symmetric and cross kernels
 * and skb_flow_set_self_exclusion apply, and its rows are bitwise those of that call.  params / v_growth / force_scale as
 * skb_flow_build_fiber_rhs; f_external 3 x N_f or NULL (no external fiber force: no fiber flow);
 * body_forces_torques 6 x n_bodies (as skb_flow_matvec) or NULL (all zero, the reference's `.any()` false).
 * Needs skb_flow_set_fiber_class and _class_derivatives for every node count in use and, with bodies,
 * skb_flow_set_body_operators (its node counts place each body's six rows); not the fiber operators, their inverse or
 * the links, and it leaves them and the body operators untouched.  Refused (SKB_ERR_INVALID, before any launch,
 * earlier state untouched): what skb_flow_build_fiber_rhs refuses, NULL params or rhs where there are fibers or
 * entries, a non-finite external force or torque (host forms: the _device form does not read its inputs on the host),
 * bodies without body operators, a group member, a target window or ranges that do not cover every row (over several
 * devices use skb_mflow_build_system_rhs, or on one process per GPU skb_flow_group_build_system_rhs_device).
 * The _device form follows skb_flow_build_fiber_rhs_device: everything on this flow's device, asynchronous on `stream`,
 * the per-fiber tables from host memory; d_body_forces / d_body_torques 3 x n_bodies each (as skb_flow_matvec_device),
 * either NULL for zero. */
SKB_API int skb_flow_build_system_rhs(skb_flow *fl, const skb_fiber_params *params, const double *v_growth,
                                      const double *force_scale, const double *f_external,
                                      const double *body_forces_torques, double dt, double eta, double *rhs);
SKB_API int skb_flow_build_system_rhs_device(skb_flow *fl, const skb_fiber_params *params, const double *v_growth,
                                             const double *force_scale, const double *d_f_external,
                                             const double *d_body_forces, const double *d_body_torques, double dt,
                                             double eta, double *d_rhs, void *stream);

/* ---- the solve of the whole system ----------------------------------------------------------------------------------
 * Solver::solve (solver_hydro.cpp:64-95) as the reference configures Belos: restarted GMRES with right preconditioning
 * (each Arnoldi step is z = P^-1 v_k, then w = A z, with the two system calls above), x0 = 0 (Solver's X_ is a fresh zero
 * vector at every System::solve), ICGS orthogonalization (two classical Gram-Schmidt passes, then the normalization), the
 * Hessenberg least-squares problem by Givens rotations on the host.  The implicit residual estimate |g_{k+1}| ends a cycle
 * once it is <= tol ||b||_2; then x += P^-1 V y and the explicit ||b - A x||_2 decides: <= tol ||b||_2 is convergence,
 * anything else restarts from x (never convergence on the implicit estimate alone).  A cycle also ends after num_blocks
 * steps (a restart from x) and at max_iters Arnoldi steps in all (converged = 0 unless the explicit residual then meets
 * tol; the current iterate is returned, SKB_OK).  A new vector whose norm after the two passes is 0 or at most
 * 16 u (u = 2^-53) of its norm before them spans nothing new ("happy breakdown"): the Krylov space is invariant, the
 * step is taken as an exact solve in it, and the explicit check follows.  ||b|| = 0: x = 0, converged, 0 iterations.
 * Belos's defaults, which the reference keeps: Num Blocks 300, Maximum Iterations 1000; gmres_tol defaults to 1e-10.
 *
 * The basis V stays on the device (column-major, num_blocks + 1 columns); one Arnoldi step is three passes over it
 * (DESIGN.md §3.8), every dot summed in a fixed order without atomics, so a solve is bitwise reproducible run to run.
 * After each step the Hessenberg column goes to pinned host memory with one event wait: the call is asynchronous on
 * `stream` except for that wait per step and one per cycle end.
 *
 * skb_flow_set_gmres: sizes the workspace for the flow's current solution size and up to num_blocks basis vectors per
 *   cycle ((num_blocks + 1) x n doubles for V: 971 MB at n = 403 206 and 300 blocks).  Call it after the set-up that
 *   fixes the solution size (skb_flow_set_fibers / _periphery / _bodies / skb_flow_set_body_operators), and again when it
 *   changes.  Refused: num_blocks outside [1, SKB_GMRES_MAX_BLOCKS].
 * skb_flow_solve_system(_device): x = A^-1 rhs on whole solution vectors (the layout of skb_flow_apply_system_matvec);
 *   dn holds SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY and SKB_DENSE_M_INV (NULL only without periphery).  info is filled
 *   on SKB_OK; history, if not NULL, holds max_iters + 1 doubles and receives the implicit relative residual after each
 *   of the info->iterations steps (history[0] = 1, the start x0 = 0).  The host form ships rhs once and x once; the
 *   _device form takes both on the flow's device.  Refused (SKB_ERR_INVALID, before any launch, x and earlier state
 *   untouched): everything skb_flow_apply_system_matvec and _preconditioner refuse, eta <= 0, tol <= 0 or not finite,
 *   num_blocks outside [1, the num_blocks of skb_flow_set_gmres], max_iters < 0, NULL info, no skb_flow_set_gmres for
 *   the current solution size.  A solution vector of length 0 returns SKB_OK (converged, 0 iterations) without a
 *   launch or a workspace. */
#define SKB_GMRES_MAX_BLOCKS 1024
typedef struct skb_solve_info {
    int32_t converged;        /* 1: ||b - A x||_2 <= tol ||b||_2 */
    int32_t iterations;       /* Arnoldi steps in all */
    int32_t restarts;         /* cycles after the first */
    int32_t reserved;
    double implicit_residual; /* the last implicit estimate |g_{k+1}| / ||b||_2 */
    double explicit_residual; /* ||b - A x||_2 / ||b||_2 of the returned x (0 when ||b|| = 0) */
    double residual;          /* ||b - A x||_2, what Solver::get_residual logs */
} skb_solve_info;
SKB_API int skb_flow_set_gmres(skb_flow *fl, int num_blocks);
SKB_API int skb_flow_solve_system(skb_flow *fl, struct skb_dense *dn, const double *rhs, double eta, double tol,
                                  int num_blocks, int max_iters, double *x, skb_solve_info *info, double *history);
SKB_API int skb_flow_solve_system_device(skb_flow *fl, struct skb_dense *dn, const double *d_rhs, double eta,
                                         double tol, int num_blocks, int max_iters, double *d_x, skb_solve_info *info,
                                         double *history, void *stream);
/* One rank per GPU (the local-vector calls below): skb_flow_set_gmres on a group member sizes the workspace for its
 * LOCAL rows (after skb_flow_group_set_body_operators, which lays them out); skb_flow_group_solve_system_device solves
 * on the local vectors d_rhs_local / d_x_local, with A and P^-1 the member's skb_flow_group_apply_system_matvec_device
 * (dn_spc: its rows of SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY) and _preconditioner_device (dn_minv: its rows of
 * SKB_DENSE_M_INV).  Every dot product is an all-reduce over the members through the group window (DESIGN.md §4): each
 * member adds every member's partial sums in rank order, so all of them hold bitwise the same Hessenberg column, take
 * the same decisions and stop at the same step, and return bitwise the same info and history.  A member that owns no
 * row takes part all the same (its vectors may be NULL).  Every member must call it with the same tol, num_blocks and
 * max_iters; a refusal is local to the rank (as for the other group calls: agree on the set-up's return codes first).
 * Refused besides what skb_flow_solve_system refuses: what the two local-vector calls refuse, a workspace set up for
 * other target ranges.  On a flow that is no member: skb_flow_solve_system_device (dn_spc and dn_minv may be one handle
 * holding both). */
SKB_API int skb_flow_group_solve_system_device(skb_flow *fl, struct skb_dense *dn_spc, struct skb_dense *dn_minv,
                                               const double *d_rhs_local, double eta, double tol, int num_blocks,
                                               int max_iters, double *d_x_local, skb_solve_info *info,
                                               double *history, void *stream);

/* ---- one timestep of the whole system ----------------------------------------------------------------------------
 * System::step (system.cpp:482-492) on a single-device flow, in the reference's order (DESIGN.md §3.9):
 *   1. skb_flow_set_fiber_links from the current placement: site = c + R(q) site_ref of each bound fiber, its bending
 *      rigidity from params;
 *   2. skb_flow_build_fiber_operators(params, dt, eta);
 *   3. skb_flow_build_system_rhs_device (params, v_growth, force_scale, f_external, body_forces_torques);
 *   4. skb_flow_solve_system_device from x0 = 0 into the workspace of skb_flow_set_gmres;
 *   5. the fiber step kernel: FiberContainerFiniteDifference::step (fcfd.cpp:292-302), ::repin_to_bodies (:308-316) to
 *      the nucleation sites at the bodies' new placement, and ::fiber_error_local (:79-89) on the repinned nodes;
 *   6. the bodies' step on the host from their rows [U; w] (48 bytes per body): c_new = c + dt U, phi = dt w and, if
 *      |phi| > 0, q_new = (cos |phi|/2, sin(|phi|/2) phi/|phi|) * q (Eigen's product order), normalised;
 *   7. the new geometry installed: the fiber positions through skb_flow_set_fibers (node counts and lengths unchanged),
 *      the bodies through skb_flow_place_bodies(c_new, q_new), the links at the new sites.
 * The step is not refused for a solve that did not converge: it advances from whatever the solve returned, as the
 * reference does, and info->solve reports it.  x (the solution, NULL ok) and tension (N_f, NULL ok) receive the step's
 * solution.  info->fiber_error is the max over fibers and nodes of | ||xs_i|| - 1 | after the step (0 without fibers),
 * info->worst_fiber the first fiber attaining it (-1 without fibers).
 *   fiber_body: per fiber its body (binding_site_.first, -1 free; NULL: all free); site_ref: 3 per fiber, the body-frame
 *   nucleation site (nucleation_sites_ref_ of the binding site; NULL without bound fibers).  Bodies must be placed by
 *   skb_flow_set_body_frames (with A_inv0) and a first skb_flow_place_bodies: the step places from the frames.
 * Two deviations from the reference (DESIGN.md §5): a body always moves to c + dt U (the reference translates only
 * inside place(), which it calls only when |phi| != 0), and q_new is normalised (placement refuses a quaternion that
 * drifted off unit norm).  A solution whose new fiber positions or body rows are not finite is not installed: geometry
 * and placement stay, info->fiber_error is NaN and the call returns SKB_ERR_STATE.
 * Refused (SKB_ERR_INVALID, before any launch, earlier state untouched): everything the four composed calls refuse,
 * dt <= 0 or not finite, bodies without frames and a first placement, a fiber_body index outside [-1, n_bodies), a
 * group member, a target window or ranges that do not cover every row, no skb_flow_set_gmres for the current solution
 * size (which also sizes the step's own buffers; the composed calls size theirs on their first use, as they do when
 * called alone).  An empty block needs none of its
 * set-up; an empty system returns SKB_OK (converged, nothing moves) without a launch.
 * skb_flow_fiber_error: the step kernel's error on the current geometry: *max_error over every fiber, per_fiber (NULL
 *   ok) per fiber.  Needs skb_flow_set_fiber_class of every node count, n <= 128.
 * skb_flow_get_placement: the centres (3 per body) and quaternions (4 per body) of the last skb_flow_place_bodies (or
 *   step); NULL skips an array.  Refused when the bodies were not placed since skb_flow_set_bodies.
 * skb_flow_get_fibers: the fiber positions (3 x N_f) of the last skb_flow_set_fibers (or step), from the host copy the
 *   flow keeps. */
typedef struct skb_step_info {
    skb_solve_info solve; /* as skb_flow_solve_system */
    double fiber_error;   /* max over fibers and nodes after the step; 0 without fibers; NaN: not installed */
    int32_t worst_fiber;  /* the fiber attaining it, -1 without fibers */
    int32_t collided;     /* System::check_collision of the installed geometry (skb_flow_set_periphery_shape); 0
                             without a shape or when the step was not installed */
} skb_step_info;
SKB_API int skb_flow_step(skb_flow *fl, struct skb_dense *dn, const skb_fiber_params *params, const double *v_growth,
                          const double *force_scale, const double *f_external, const double *body_forces_torques,
                          const int *fiber_body, const double *site_ref, double dt, double eta, double tol,
                          int num_blocks, int max_iters, double *x, double *tension, skb_step_info *info);
SKB_API int skb_flow_fiber_error(skb_flow *fl, double *max_error, double *per_fiber);
/* skb_flow_step on one rank per GPU, on a connected group member (the local-vector calls below).  params, v_growth,
 * force_scale, fiber_body and site_ref cover the OWN fibers (as skb_flow_group_set_fiber_links); d_f_external holds 3
 * values per own fiber node, d_body_forces / d_body_torques 3 per body of ALL bodies (each NULL ok), all on the device;
 * dn_spc / dn_minv are the member's row blocks of the two periphery operators.  In order:
 *   1. skb_flow_group_set_fiber_links from the current placement, skb_flow_build_fiber_operators,
 *      skb_flow_group_build_system_rhs_device and skb_flow_group_solve_system_device: the solution is bitwise what a
 *      caller composing those calls gets;
 *   2. the body rows all-gathered through the group window (an epoch of its own): every member reads [U; w] of every
 *      body from its own window and steps the bodies on the host, so all hold the same placement and sites;
 *   3. the step kernel over the own fibers, its new positions and per-fiber errors stored straight into every member's
 *      window (an epoch of its own); every member reads the complete positions and errors from its own window;
 *   4. the non-finite checks and the error's max over the COMPLETE arrays: every member returns the same code,
 *      fiber_error and worst_fiber (a fiber index among ALL fibers); a non-finite solution is installed by no member
 *      (SKB_ERR_STATE, NaN fiber_error);
 *   5. the install: skb_flow_set_fibers with the complete positions, skb_flow_group_place_bodies, and
 *      skb_flow_group_set_fiber_links at the new sites.
 * d_x_local (NULL ok) receives the member's local rows of the solution, d_tension (NULL ok) the tension of its own
 * fiber nodes.  The call runs on `stream` (the links, the build and the install on the flow's own stream, drained
 * before it returns).  It allocates no device memory and loads no kernel: skb_flow_set_gmres on the member, called
 * after the fiber classes and their derivatives are set, sizes and loads what it uses -- the step's buffers, the fiber
 * build's and the fiber-body links' for the own fibers, and a pinned host copy through which the device inputs' finiteness
 * is checked (DESIGN.md §3.9).  Every member must call it alike.  Refused, locally and before any launch: what
 * skb_flow_step refuses (but for membership and the whole target list; f_external and the body forces and torques are
 * read back for their check), what the local-vector calls refuse, no skb_flow_set_gmres for the member's current target
 * ranges or none since the fiber classes were set, a fiber_body index outside [-1, n_bodies) among the own fibers.  On a flow that is no group member: skb_flow_step, its x and tension on the device (dn_spc holds both
 * operators; dn_minv is not read). */
SKB_API int skb_flow_group_step_device(skb_flow *fl, struct skb_dense *dn_spc, struct skb_dense *dn_minv,
                                       const skb_fiber_params *params, const double *v_growth,
                                       const double *force_scale, const double *d_f_external,
                                       const double *d_body_forces, const double *d_body_torques,
                                       const int *fiber_body, const double *site_ref, double dt, double eta,
                                       double tol, int num_blocks, int max_iters, double *d_x_local,
                                       double *d_tension, skb_step_info *info, void *stream);
SKB_API int skb_flow_get_placement(skb_flow *fl, double *centers, double *orientations);
SKB_API int skb_flow_get_fibers(skb_flow *fl, double *r_fib);

/* ---- the periphery's shape: repulsion, binding and collision inside the step --------------------------------------
 * What System::prep_state_for_solver and System::run do with the periphery's shape besides its operators, on the
 * device (DESIGN.md §3.9): fc_->periphery_force (system.cpp:422; SphericalPeriphery / EllipsoidalPeriphery::
 * fiber_interaction, periphery.cpp:140-162, 232-263), fc_->update_boundary_conditions (system.cpp:452,
 * fiber_finite_difference.cpp:74-91) and System::check_collision (system.cpp:576-595).
 *   repulsion of node i strictly inside the surface (|x| < R, or |x| < |r_cortex| with the reference's 1e-12 guards in
 *     atan2 and acos): f_0 dr / |dr| exp(-(R - |x|) / l_0), dr = x - (the surface point in the direction of x); 0 on
 *     or outside the surface and at node 0 of a fiber with fiber_minus_clamped.  A node at the exact centre of a
 *     sphere divides 0 by 0 as the reference does: its force is NaN (a step refuses it, below).
 *   plus_hinged of a fiber = binding_active && polar_angle_start <= acos(normalized(x_last).z) <= polar_angle_end &&
 *     some node within binding_threshold of the surface (normalized() of a zero vector is zero: angle pi/2).
 *   collided = a fiber node on or beyond the surface (node 0 skipped when the fiber is minus-clamped: params
 *     minus_clamped of the last step, fiber_minus_clamped before one), a spherical body with |c| + r > R (sphere
 *     only), or two spherical bodies with |c1 - c2| < r1 + r2.
 * With a shape set, skb_flow_step, skb_flow_group_step_device and skb_mflow_step (on every member):
 *   1. before the links and the fiber build, run the pass on the current geometry (own fibers); a non-finite
 *      repulsion is refused there (SKB_ERR_INVALID, geometry untouched), as a non-finite f_external is;
 *   2. step with f_external + repulsion (the repulsion alone for a NULL f_external), and with every stepped fiber's
 *      params plus_hinged replaced by the pass's value -- the reference sets bc_plus_ of every fiber every step, so
 *      the caller's plus_hinged is ignored then;
 *   3. after the install, run the pass over ALL fibers and bodies and set info->collided.  Every member of a group
 *      holds the complete new geometry and returns the same value: each member's own fibers' params minus_clamped
 *      travel with their new positions in the step's all-gather, so every member skips node 0 of the same fibers.
 *      A step that is refused or not installed leaves the flags the collision test uses as they were.
 * skb_flow_set_periphery_shape: the shape, fiber_minus_clamped (per fiber the TOML flag minus_clamped_, not
 *   is_minus_clamped(); NULL: all 0) and body_radius (per body the radius of a spherical body, 0: not spherical, never
 *   colliding; NULL: no body takes part).  Sizes the pass's buffers (with a pinned flag buffer) for the flow's fibers
 *   and loads its kernels; skb_flow_set_gmres sizes them again.  SKB_PERIPHERY_NONE clears the shape (the reference's
 *   GenericPeriphery: no force, no binding, no collision).  Refused (SKB_ERR_INVALID, before any launch, the earlier
 *   shape kept): a kind outside the enum, a non-finite parameter, a, b or c <= 0 for the kind in use (a alone for a
 *   sphere), l_0 <= 0, a flag outside {0, 1}, a negative or non-finite radius, a flow without periphery nodes.  A step
 *   is refused when the flow's fibers or bodies changed in number since the call (call it again), or when its nodes
 *   outgrew the buffers (skb_flow_set_gmres sizes them again).
 *   Every member of a group makes the same call with the complete arrays.
 * skb_flow_periphery_interaction: the pass on the current geometry: f_periphery 3 per own node, plus_hinged per own
 *   fiber, *collided over ALL fibers and bodies; each output may be NULL.  Refused without a shape. */
enum { SKB_PERIPHERY_NONE = 0, SKB_PERIPHERY_SPHERE = 1, SKB_PERIPHERY_ELLIPSOID = 2 };
typedef struct skb_periphery_shape {
    int32_t kind;           /* SKB_PERIPHERY_*; NONE also stands for the reference's GenericPeriphery          */
    int32_t binding_active; /* periphery_binding.active                                                        */
    double a, b, c;         /* SphericalPeriphery::radius_ (a; b, c ignored) / EllipsoidalPeriphery a_, b_, c_ */
    double f_0, l_0;        /* fiber_periphery_interaction (params.hpp:45-48)                                  */
    double polar_angle_start, polar_angle_end, binding_threshold; /* periphery_binding (params.hpp:25-29)    */
} skb_periphery_shape;
SKB_API int skb_flow_set_periphery_shape(skb_flow *fl, const skb_periphery_shape *shape,
                                         const int32_t *fiber_minus_clamped, const double *body_radius);
SKB_API int skb_flow_periphery_interaction(skb_flow *fl, double *f_periphery, int32_t *plus_hinged,
                                           int32_t *collided);

/* ---- dynamic instability: catastrophe, growth and nucleation before each step --------------------------------------
 * System::dynamic_instability (dynamic_instability.cpp:25-194), the first statement of System::prep_state_for_solver,
 * on a single-device flow (DESIGN.md §3.11).  di.n_nodes == 0 changes nothing (the reference's early return).  Else,
 * for each fiber f in container order, pinned = plus_pinned[f]:
 *   v = v_growth, fc = f_catastrophe, each times its *_collision_scale when pinned;
 *   the fiber is removed when u_f > exp(-dt fc) (u_f the draw (f, 0) of the stream below);
 *   a survivor gets length_prev = length, length = length + dt v (v_growth_out = v); a bound survivor occupies its site.
 * Then n_new = min(Poisson(dt nucleation_rate (n_sites - fibers bound before the catastrophe)), free sites), the sites
 * picked uniformly without replacement (a partial Fisher-Yates over the free flat sites in ascending order), and one
 * new fiber per pick appended after the survivors in pick order: di.n_nodes nodes, length = length_prev = min_length,
 * radius, bending_rigidity, penalty_param 500, beta_tstep 1, minus_clamped 1, plus_hinged 0, v_growth 0, a straight
 * line from the site (c + R(q) site_ref at the current placement) along (site - c) / |site - c|.
 * The draws come from Philox4x32-10 with key = seed and counter = (i, purpose, call counter): the result depends on
 * (seed, counter) and the inputs only.  It is not the reference's stream (DESIGN.md §5).
 *   skb_flow_set_nucleation_sites: the bodies' nucleation_sites_ref_ (body frame), once per run: n_sites_per_body per
 *     body of skb_flow_set_bodies, site_ref 3 per site, bodies concatenated.  Refused: a NULL count table with bodies,
 *     a negative count, a non-finite site or one at the body's centre.
 *   skb_flow_dynamic_instability: n_in == the flow's fiber count; params_in, binding_in ((body, site) per fiber, -1 for
 *     a free fiber), plus_pinned (bc_plus_ of the last step: skb_flow_step_flags, or the caller's at the start) per
 *     input fiber.  The outputs hold `capacity` fibers: *n_out, params_out, binding_out, v_growth_out and origin_out
 *     (the input fiber output fiber f came from, -1 for a nucleated one: through it the caller carries its own
 *     per-fiber arrays, such as force_scale).  On SKB_OK the flow holds the new fibers -- positions, node counts and
 *     lengths through the skb_flow_set_fibers path, the periphery shape's per-fiber flags carried through origin (0
 *     for new fibers) and its buffers sized, the GMRES workspace and the step's buffers sized at the num_blocks of the
 *     last skb_flow_set_gmres -- and the next skb_flow_step needs no other set-up.  Refused (SKB_ERR_INVALID, before
 *     any launch, the geometry untouched): a group member (its window is sized for a fixed fiber set), dt <= 0 or not
 *     finite, a non-finite or negative rate or scale, a non-positive min_length or radius, a negative bending rigidity,
 *     di.n_nodes outside [8, 128] or without skb_flow_set_fiber_class and _class_derivatives, a binding outside the
 *     sites, a plus_pinned outside {0, 1}, bodies without sites or placement, n_in != the flow's fiber count,
 *     capacity < n_in + the number of sites.  skb_mflow has no such call.
 *   skb_flow_step_flags: plus_hinged of each fiber as the last installed skb_flow_step built it (the periphery
 *     binding's value with a shape, the caller's otherwise): bc_plus_ at the next is_plus_pinned().  Carried through
 *     skb_flow_dynamic_instability (0 for new fibers).  Refused when no step was installed for the current fiber count. */
typedef struct skb_dynamic_instability { /* params.hpp:30-42 (min_separation is never used there) */
    int32_t n_nodes;                     /* nodes of a nucleated fiber; 0: the model is off */
    int32_t reserved;
    double v_growth, f_catastrophe, v_grow_collision_scale, f_catastrophe_collision_scale, nucleation_rate;
    double radius, min_length, bending_rigidity;
} skb_dynamic_instability;
typedef struct skb_dynamic_info {
    int32_t removed, nucleated, grown, reserved;
    double mu; /* the Poisson mean of the nucleation count */
} skb_dynamic_info;
SKB_API int skb_flow_set_nucleation_sites(skb_flow *fl, const int *n_sites_per_body, const double *site_ref);
SKB_API int skb_flow_dynamic_instability(skb_flow *fl, const skb_dynamic_instability *di, double dt, uint64_t seed,
                                         uint64_t counter, int n_in, const skb_fiber_params *params_in,
                                         const int32_t *binding_in, const int32_t *plus_pinned, int capacity,
                                         int *n_out, skb_fiber_params *params_out, int32_t *binding_out,
                                         double *v_growth_out, int32_t *origin_out, skb_dynamic_info *info);
SKB_API int skb_flow_step_flags(skb_flow *fl, int32_t *plus_hinged);

/* ---- the whole-vector calls on one rank per GPU ---------------------------------------------------------------------
 * A group member (skb_flow_group_init ... skb_flow_group_warmup above) applies A, P^-1 and builds the RHS on its LOCAL
 * vector: its own rows of the whole vector [fibers | shell | bodies], in ascending global order --
 *   x_local = [4 per own fiber node | 3 per own periphery row | own body rows],
 * the own body rows being the 3 rows of each body node in its body rows [b0, b1) (skb_flow_set_target_ranges) and the
 * six rows [U; w] of every body whose FIRST node lies in [b0, b1) (the rows of skb_mflow_apply_system_matvec,
 * distributed.system_rows; skb_group_body_pieces gives their places).  The members' local vectors tile the whole vector
 * once; no rank needs a full-length vector.  Every member stores its own body rows (for the preconditioner also its own
 * periphery rows) into all windows and meets its peers at a flag before it reads the complete x_bodies / x_shell from
 * its own window; the rest is the protocol of skb_mflow, and the results are bitwise those of skb_mflow on the same
 * device list.
 *   skb_flow_group_set_body_operators: the arrays of ALL bodies, as skb_flow_set_body_operators (bodies are complete on
 *     every member); the member keeps the inverses of the bodies it owns rows of, lays out its body rows, and sizes every
 *     buffer the three calls below use, for the member's current target ranges (all six of them).  After
 *     skb_flow_group_init and the target ranges; a change of the ranges wants the group set up again (init, the
 *     handle exchange, the warm-up) and then this call, or the three calls below refuse.
 *   skb_flow_group_set_fiber_links: body / site / bending_rigidity of the OWN fibers (as every per-fiber array under
 *     target ranges), otherwise as skb_flow_set_fiber_links.
 *   skb_flow_group_apply_system_matvec_device: d_res_local = the own rows of A x; dn holds the member's rows of
 *     SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY (3 n_own_shell x 3 N_s, skb_dense_create_on this flow's device; may be
 *     NULL without own periphery rows).
 *   skb_flow_group_apply_system_preconditioner_device: d_y_local = the own rows of P^-1 x; dn holds the member's rows of
 *     SKB_DENSE_M_INV.
 *   skb_flow_group_build_system_rhs_device: d_rhs_local = the own rows of the RHS; params / v_growth / force_scale of
 *     the OWN fibers, d_f_external 3 per own fiber node or NULL, d_body_forces / d_body_torques complete (3 x n_bodies
 *     each, as skb_flow_build_system_rhs_device) or NULL: they enter the body flow as they are, once.
 * All three are asynchronous on `stream`; consecutive calls of a member must be ordered (one stream, or the caller's
 * events).  Every member must make the same sequence of calls, as with any collective.  A refusal (SKB_ERR_INVALID /
 * SKB_ERR_STATE, before any launch, earlier state untouched) is LOCAL to the rank that refused: the refusals of the
 * single-device twins, a dense block that does not fit the member's rows and the current periphery, no
 * skb_flow_group_set_body_operators for the member's current target ranges (fiber, periphery AND body rows), a member whose peers are not all
 * connected.  A rank that goes on after a peer refused waits on a flag until the time-out (skb_flow_group_error), so a
 * caller agrees on the set-up calls' return codes (e.g. an all-reduce) before the first apply.  None of the three
 * allocates device memory: the set-up calls and the warm-up sized everything, so no cudaMalloc / cudaFree meets a
 * peer's flag wait on the same device.  On a flow that is not a group member the five calls are the single-device
 * calls (whole vector, bitwise). */
SKB_API int skb_flow_group_set_body_operators(skb_flow *fl, const int *n_nodes, int n_bodies,
                                              const double *node_weights, const double *ex, const double *ey,
                                              const double *ez, const double *A_inv);
SKB_API int skb_flow_group_set_fiber_links(skb_flow *fl, const int *body, const double *site,
                                           const double *bending_rigidity);
/* skb_flow_set_body_frames / _place_bodies on a group member (arrays of ALL bodies).  The frames call also does what
 * skb_flow_group_set_body_operators does: the member keeps the body-frame inverses of the bodies it owns rows of,
 * lays out its body rows and sizes every buffer, the placement's included.  The place call then allocates no device
 * memory and loads no kernel, so it may run while a peer on the same device waits on a flag; it refuses, locally, what
 * skb_flow_place_bodies refuses and body rows other than the frames'.  Not a member: the single-device calls. */
SKB_API int skb_flow_group_set_body_frames(skb_flow *fl, const int *n_nodes, int n_bodies, const double *node_pos_ref,
                                           const double *node_normal_ref, const double *node_weights,
                                           const double *ex0, const double *ey0, const double *ez0,
                                           const double *A_inv0);
SKB_API int skb_flow_group_place_bodies(skb_flow *fl, const double *centers, const double *orientations);
SKB_API int skb_flow_group_apply_system_matvec_device(skb_flow *fl, struct skb_dense *dn, const double *d_x_local,
                                                      double eta, double *d_res_local, void *stream);
SKB_API int skb_flow_group_apply_system_preconditioner_device(skb_flow *fl, struct skb_dense *dn,
                                                              const double *d_x_local, double *d_y_local,
                                                              void *stream);
SKB_API int skb_flow_group_build_system_rhs_device(skb_flow *fl, const skb_fiber_params *params,
                                                   const double *v_growth, const double *force_scale,
                                                   const double *d_f_external, const double *d_body_forces,
                                                   const double *d_body_torques, double dt, double eta,
                                                   double *d_rhs_local, void *stream);
/* host-only (no GPU needed): the places of a member's own body rows [body_begin, body_end) -- as runs of consecutive
 * entries, 3 int64 per run: offset in the local vector's body part, offset in the whole vector's body part, length.
 * *n_pieces = the number of runs (at most 3); refused if it exceeds max_pieces. */
SKB_API int skb_group_body_pieces(const int *n_nodes, int n_bodies, int64_t body_begin, int64_t body_end,
                                  int64_t *pieces, int max_pieces, int *n_pieces);

typedef struct skb_flow_stats {
    double device_ms;   /* CUDA-event time of the last call, first launch to last kernel (copies excluded) */
    double total_ms;    /* including H2D / D2H */
    int64_t n_pairs;    /* source x target pairs evaluated by the pair kernels */
    int32_t launches;
} skb_flow_stats;
SKB_API int skb_flow_last_stats(const skb_flow *fl, skb_flow_stats *out);
/* the matvec's dominant kernel (symmetric fiber-fiber block): duration of its last launch and the ordered pairs it
 * covered (skb_ctx_last_sym_kernel of the matvec's fiber evaluator) -- the roofline line of bench.py */
SKB_API int skb_flow_last_sym_kernel(const skb_flow *fl, double *ms, int64_t *pairs);

/* ---- skb_mflow: ONE process driving n GPUs ---------------------------------------------------------------------
 * The multi-device form the reference's rule "direct evaluators need a single MPI rank" (system.cpp:618-623) admits.
 * Same calls and array conventions as skb_flow, complete host arrays in and out; internally one group member per
 * device (see the group section above), each driven by its own host thread.  Whole fibers (balanced by node count),
 * periphery rows and body rows are block-partitioned over the devices; the periphery's dense operators are stored by
 * row blocks (periphery.cpp:387-417).  devices == NULL: 0..n-1.  (A device may be listed more than once: that
 * exercises the exchange protocol on a single GPU and is meant for tests.) */
typedef struct skb_mflow skb_mflow;
SKB_API int skb_mflow_create(const int *devices, int n, skb_mflow **out);
SKB_API int skb_mflow_destroy(skb_mflow *mf);
SKB_API int skb_mflow_n_devices(const skb_mflow *mf, int *n);
SKB_API int skb_mflow_set_fibers(skb_mflow *mf, const double *r_fib, const int *n_nodes, const double *length,
                                 int n_fibers);
SKB_API int skb_mflow_set_periphery(skb_mflow *mf, const double *node_pos, const double *node_normal, int64_t n_nodes);
SKB_API int skb_mflow_set_bodies(skb_mflow *mf, const double *node_pos, const double *node_normal, int64_t n_nodes,
                                 const double *centers, int n_bodies);
SKB_API int skb_mflow_set_self_exclusion(skb_mflow *mf, int fused);
SKB_API int skb_mflow_set_cross(skb_mflow *mf, int mode);
SKB_API int skb_mflow_set_overlap(skb_mflow *mf, int on); /* skb_flow_set_overlap on every member */
/* which fibers / periphery rows / body rows device `member` owns (any pointer may be NULL) */
SKB_API int skb_mflow_partition(skb_mflow *mf, int member, int *fiber_begin, int *fiber_end, int64_t *shell_begin,
                                int64_t *shell_end, int64_t *body_begin, int64_t *body_end);
/* the same partition without a GPU or a handle (rank-per-GPU hosts): out6 = the six arguments of
 * skb_flow_set_target_ranges for `member` of `n_members` */
SKB_API int skb_partition_query(const int *n_nodes, int n_fibers, int64_t n_shell, int64_t n_body, int n_members,
                                int member, int64_t *out6);
SKB_API int skb_mflow_set_fiber_class(skb_mflow *mf, int n_nodes, const double *D_1_0, const double *P_downsample_bc);
/* complete arrays of ALL fibers, as skb_flow_set_fiber_operators without a window; every device keeps its own slice */
SKB_API int skb_mflow_set_fiber_operators(skb_mflow *mf, const double *A, const double *force_operator,
                                          const double *xs, const double *length_prev, const int *plus_bc_velocity);
SKB_API int skb_mflow_set_fiber_preconditioner(skb_mflow *mf, const double *A_inv);
SKB_API int skb_mflow_set_fiber_class_derivatives(skb_mflow *mf, int n_nodes, const double *D_2_0,
                                                  const double *D_3_0, const double *D_4_0);
/* params of ALL fibers; every member builds its own slice on its own device, in parallel */
SKB_API int skb_mflow_build_fiber_operators(skb_mflow *mf, const skb_fiber_params *params, double dt, double eta);
/* skb_flow_build_fiber_rhs with the complete arrays of ALL fibers; every member forms its own slice of rhs */
SKB_API int skb_mflow_build_fiber_rhs(skb_mflow *mf, const skb_fiber_params *params, const double *v_growth,
                                      const double *force_scale, const double *v_on_fibers, const double *f_external,
                                      double dt, double eta, double *rhs);
/* op = skb_dense_op (skelly_b200_dense.h); A row-major (3 N_s) x (3 N_s) */
SKB_API int skb_mflow_set_dense(skb_mflow *mf, int op, const double *A_rowmajor, int64_t n_rows, int64_t n_cols);
SKB_API int skb_mflow_matvec(skb_mflow *mf, const double *fib_forces, const double *shell_density,
                             const double *body_densities, const double *body_forces_torques, double eta,
                             double *v_all);
/* out_shell = res_shell when skb_mflow_set_dense(SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY, ...) was called, else v_shell */
SKB_API int skb_mflow_apply_matvec(skb_mflow *mf, const double *x_fibers, const double *x_shell,
                                   const double *body_densities, const double *body_forces_torques,
                                   const double *fiber_link_conditions, double eta, double *res_fibers,
                                   double *out_shell, double *v_bodies);
/* The whole-vector operator and preconditioner over n devices: the skb_flow_set_body_operators / _set_fiber_links /
 * _apply_system_matvec / _apply_system_preconditioner twins, with the same arguments (complete host arrays of all
 * bodies and all fibers, the whole solution vector in and out), the same refusals (before any launch, earlier state
 * untouched; the body checks cover every body and fiber, not just a member's) and the same drop rules
 * (skb_mflow_set_bodies drops the body operators and the links, skb_mflow_set_fibers / _set_fiber_class the links).
 * The periphery's operators come from skb_mflow_set_dense: SKB_DENSE_STRESSLET_PLUS_COMPLEMENTARY for the matvec,
 * SKB_DENSE_M_INV for the preconditioner; each member's row block must fit the current periphery (after
 * skb_mflow_set_periphery changed the node count, a block set before is refused until skb_mflow_set_dense is called
 * again).  A change of the number of bodies re-initialises the group (its window carries the link forces): the fiber
 * operators must then be set again, as after any change of the node counts.
 *   Rows: member g owns, besides its fibers' and periphery rows (skb_mflow_partition), the 3 rows of each body node in
 * its body rows [b0, b1) and the six rows [U; w] of every body whose FIRST node lies in [b0, b1); it keeps the
 * inverses of the bodies it owns rows of.  x_bodies is complete on every member (system.cpp:306-311), so a body's
 * K^T lambda sums over all of its nodes wherever its six rows are.
 *   Link forces: every member computes the link conditions of its own fibers and, per body, the sum of its own bound
 * fibers' forces and torques in container order; the members' partials are exchanged through the group window and
 * added in member (rank) order, 0 first (the MPI_Allreduce of body_container.cpp:128-135).  Every member thus holds
 * bitwise the same totals, and the result is bitwise reproducible run to run for a given device list; it differs from
 * the single-device order by rounding only.
 *   Each member runs the rank-per-GPU calls (skb_flow_group_set_body_operators / _set_fiber_links on its own fibers'
 * slices, skb_flow_group_apply_system_matvec_device / _preconditioner_device on its local rows, which the driver
 * gathers from and scatters into the whole host vector).  A member's rows are laid out again before a system call
 * whenever a new partition re-initialised the group, so no new skb_mflow_set_body_operators is needed after one.
 * With one device it is the skb_flow path. */
SKB_API int skb_mflow_set_body_operators(skb_mflow *mf, const int *n_nodes, int n_bodies, const double *node_weights,
                                         const double *ex, const double *ey, const double *ez, const double *A_inv);
SKB_API int skb_mflow_set_fiber_links(skb_mflow *mf, const int *body, const double *site,
                                      const double *bending_rigidity);
/* skb_flow_set_body_frames / _place_bodies over n devices, forwarded to every member (each keeps the body-frame
 * inverses of the bodies it owns rows of); every member's refusals are checked before any member changes.  A new
 * partition (a change of the node counts) wants the frames set again. */
SKB_API int skb_mflow_set_body_frames(skb_mflow *mf, const int *n_nodes, int n_bodies, const double *node_pos_ref,
                                      const double *node_normal_ref, const double *node_weights, const double *ex0,
                                      const double *ey0, const double *ez0, const double *A_inv0);
SKB_API int skb_mflow_place_bodies(skb_mflow *mf, const double *centers, const double *orientations);
SKB_API int skb_mflow_apply_system_matvec(skb_mflow *mf, const double *x, double eta, double *res);
SKB_API int skb_mflow_apply_system_preconditioner(skb_mflow *mf, const double *x, double *y);
/* skb_flow_build_system_rhs over n devices, the same arguments (complete host arrays of all fibers and bodies, the whole
 * vector out) and refusals, every member's checked before any device starts.  Each member forms its own rows (those of
 * skb_mflow_apply_system_matvec) with skb_flow_group_build_system_rhs_device; the flow is the group's matvec flow, and
 * the complete F_T enter every member's body flow as they are.  With one device it is the skb_flow path. */
SKB_API int skb_mflow_build_system_rhs(skb_mflow *mf, const skb_fiber_params *params, const double *v_growth,
                                       const double *force_scale, const double *f_external,
                                       const double *body_forces_torques, double dt, double eta, double *rhs);
/* skb_flow_solve_system over n devices: complete host rhs in, complete host x out.  skb_mflow_set_gmres sizes every
 * member's workspace for its local rows (laid out again first if a new partition re-initialised the group since
 * skb_mflow_set_body_operators or _set_body_frames); each member thread then runs skb_flow_group_solve_system_device on
 * its rows, so every member reports bitwise the same info and history.  Refusals as skb_flow_solve_system's and
 * skb_mflow_apply_system_matvec's / _preconditioner's, every member's checked before any device starts; no
 * skb_mflow_set_gmres since the partition or the bodies' node counts changed.  With one device it is the skb_flow path,
 * bitwise. */
SKB_API int skb_mflow_set_gmres(skb_mflow *mf, int num_blocks);
SKB_API int skb_mflow_solve_system(skb_mflow *mf, const double *rhs, double eta, double tol, int num_blocks,
                                   int max_iters, double *x, skb_solve_info *info, double *history);
/* skb_flow_set_point_sources / _set_background on every device: skb_mflow_velocity_at_targets and
 * skb_mflow_build_system_rhs include them */
/* skb_flow_step over n devices: the same arguments as complete host arrays of all fibers and bodies, the same refusals
 * (every member's before any member launches) and the same deviations.  Every member runs skb_flow_group_step_device on
 * its own slice of the arguments, on its own host thread: the inputs go up once (each member's own f_external, the
 * complete body forces and torques), the body rows and the new fiber geometry are all-gathered through the members'
 * group windows, and every member takes the same decision and installs the same complete geometry and placement.
 * info->fiber_error is the max over all fibers.  x and tension come down once, each member's own rows.
 * skb_mflow_set_gmres sizes the step's buffers.  With one device it is bitwise skb_flow_step. */
SKB_API int skb_mflow_step(skb_mflow *mf, const skb_fiber_params *params, const double *v_growth,
                           const double *force_scale, const double *f_external, const double *body_forces_torques,
                           const int *fiber_body, const double *site_ref, double dt, double eta, double tol,
                           int num_blocks, int max_iters, double *x, double *tension, skb_step_info *info);
/* skb_mflow has no dynamic instability (skb_flow_dynamic_instability): its members' windows are sized for a fixed fiber
 * set at skb_flow_group_init. */
/* skb_flow_set_periphery_shape on every member (the complete arrays); skb_mflow_step applies it on every member */
SKB_API int skb_mflow_set_periphery_shape(skb_mflow *mf, const skb_periphery_shape *shape,
                                          const int32_t *fiber_minus_clamped, const double *body_radius);
/* skb_flow_periphery_interaction over the devices: the complete arrays of all fibers */
SKB_API int skb_mflow_periphery_interaction(skb_mflow *mf, double *f_periphery, int32_t *plus_hinged,
                                            int32_t *collided);
/* skb_flow_get_fibers / _get_placement of the geometry every member holds */
SKB_API int skb_mflow_get_fibers(skb_mflow *mf, double *r_fib);
SKB_API int skb_mflow_get_placement(skb_mflow *mf, double *centers, double *orientations);
SKB_API int skb_mflow_set_point_sources(skb_mflow *mf, const double *positions, const double *forces,
                                        const double *torques, int n_points);
SKB_API int skb_mflow_set_background(skb_mflow *mf, const int *components, const double *scale_factor,
                                     const double *uniform);
/* System::velocity_at_targets (system.cpp:330-384): targets block-partitioned over the devices */
SKB_API int skb_mflow_velocity_at_targets(skb_mflow *mf, const double *r_trg, int64_t n_trg, const double *fib_forces,
                                          const double *shell_density, const double *body_densities,
                                          const double *body_forces_torques, double eta, double *vel);
SKB_API int skb_mflow_last_stats(const skb_mflow *mf, skb_flow_stats *out);

#ifdef __cplusplus
}
#endif
#endif

// skelly_b200/flow.hpp -- C++ host-side mirror of the three container flows and of the hydrodynamic part of
// System::apply_matvec, on top of the C ABI in skelly_b200_flow.h.  Header-only, works with Eigen::MatrixXd or the
// minimal skelly_b200::Matrix (kernels.hpp).  Names and argument meaning follow the reference:
//
//   FiberContainerFiniteDifference::flow(r_trg, fib_forces, eta, subtract_self)   fcfd.cpp:172-214
//   Periphery::flow(r_trg, density, eta)                                           periphery.cpp:55-79
//   BodyContainer::flow(r_trg, body densities, forces_torques, eta)                body_container.cpp:269-477
//   System::apply_matvec  (v_all over [fibers | shell | bodies])                   system.cpp:284-316
//   System::velocity_at_targets                                                    system.cpp:330-384
//   FiberContainerFiniteDifference::apply_fiber_force / ::matvec                   fcfd.cpp:272-287, 216-232
//
// Every failure of the C ABI becomes std::runtime_error (caught in skelly_sim.cpp:57-64).
#pragma once
#include "../skelly_b200_dense.h"
#include "../skelly_b200_flow.h"
#include "kernels.hpp"

#include <algorithm>
#include <memory>
#include <vector>

namespace skelly_b200 {

template <class M> class FlowEngineT {
  public:
    explicit FlowEngineT(int device = 0) {
        st_ = std::make_shared<State>();
        check(skb_flow_create(device, &st_->fl), "skb_flow_create");
    }

    // ---- geometry: call after positions change (System::step), not per GMRES iteration ----
    /// r_fib: 3 x N_f node positions in container order; n_nodes / lengths per fiber
    void set_fibers(const M &r_fib, const std::vector<int> &n_nodes, const std::vector<double> &lengths) {
        if (n_nodes.size() != lengths.size())
            throw std::runtime_error("skelly_b200: n_nodes / lengths size mismatch");
        check(skb_flow_set_fibers(st_->fl, r_fib.data(), n_nodes.data(), lengths.data(), (int)n_nodes.size()),
              "skb_flow_set_fibers");
        st_->n_fib = r_fib.cols();
        st_->n_nodes = n_nodes;
    }
    void set_periphery(const M &node_pos, const M &node_normal) {
        check(skb_flow_set_periphery(st_->fl, node_pos.data(), node_normal.data(), node_pos.cols()),
              "skb_flow_set_periphery");
        st_->n_shell = node_pos.cols();
    }
    void set_bodies(const M &node_pos, const M &node_normal, const M &centers) {
        check(skb_flow_set_bodies(st_->fl, node_pos.data(), node_normal.data(), node_pos.cols(), centers.data(),
                                  (int)centers.cols()),
              "skb_flow_set_bodies");
        st_->n_body = node_pos.cols();
    }

    // ---- the reference's flow() functions ----
    M fiber_flow(const M &r_trg, const M &fib_forces, double eta, bool subtract_self = true) const {
        M vel = M::Zero(3, r_trg.cols());
        check(skb_flow_fibers(st_->fl, r_trg.data(), r_trg.cols(), fib_forces.data(), eta, subtract_self ? 1 : 0,
                              vel.data()),
              "skb_flow_fibers");
        return vel;
    }
    M periphery_flow(const M &r_trg, const M &density, double eta) const {
        M vel = M::Zero(3, r_trg.cols());
        check(skb_flow_periphery(st_->fl, r_trg.data(), r_trg.cols(), density.data(), eta, vel.data()),
              "skb_flow_periphery");
        return vel;
    }
    /// forces_torques: 6 x n_bodies (body_container.cpp:128-135)
    M body_flow(const M &r_trg, const M &densities, const M &forces_torques, double eta) const {
        M vel = M::Zero(3, r_trg.cols());
        check(skb_flow_bodies(st_->fl, r_trg.data(), r_trg.cols(), densities.data(), forces_torques.data(), eta,
                              vel.data()),
              "skb_flow_bodies");
        return vel;
    }
    /// hydrodynamic part of System::apply_matvec: 3 x (N_f + N_s + N_b), targets [fibers | shell | bodies]
    M matvec_flow(const M &fib_forces, const M &shell_density, const M &body_densities, const M &forces_torques,
                  double eta) const {
        M v = M::Zero(3, st_->n_fib + st_->n_shell + st_->n_body);
        check(skb_flow_matvec(st_->fl, fib_forces.data(), shell_density.data(), body_densities.data(),
                              forces_torques.data(), eta, v.data()),
              "skb_flow_matvec");
        return v;
    }
    M velocity_at_targets(const M &r_trg, const M &fib_forces, const M &shell_density, const M &body_densities,
                          const M &forces_torques, double eta) const {
        M vel = M::Zero(3, r_trg.cols());
        check(skb_flow_velocity_at_targets(st_->fl, r_trg.data(), r_trg.cols(), fib_forces.data(),
                                           shell_density.data(), body_densities.data(), forces_torques.data(), eta,
                                           vel.data()),
              "skb_flow_velocity_at_targets");
        return vel;
    }

    // ---- the listener (listener.cpp:86-136) on one frame ----
    /// body_velocities: 6 x n_bodies [U; omega]; body_kind 0 / 1 (sphere) / 2 (ellipsoid); body_radii 3 x n_bodies
    void set_listener_frame(const M &fib_forces, const M &shell_density, const M &body_densities,
                            const M &forces_torques, const M &body_velocities, const std::vector<int32_t> &body_kind,
                            const M &body_radii, double eta) {
        check(skb_flow_set_listener_frame(st_->fl, fib_forces.data(), shell_density.data(), body_densities.data(),
                                          forces_torques.data(), body_velocities.data(), body_kind.data(),
                                          body_radii.data(), eta),
              "skb_flow_set_listener_frame");
    }
    /// the frame of the installed geometry and a step's solution x (tension: N_f values), as the reference's listener
    /// unpacks a trajectory frame; leaves the fiber operators of the installed geometry resident, without their inverse
    void set_listener_state(const std::vector<skb_fiber_params> &params, double dt, double eta,
                            const std::vector<double> &tension, const std::vector<double> &x,
                            const std::vector<int32_t> &body_kind, const M &body_radii, bool periphery_interaction) {
        check(skb_flow_set_listener_state(st_->fl, params.data(), dt, eta, tension.data(), x.data(), body_kind.data(),
                                          body_radii.data(), periphery_interaction ? 1 : 0),
              "skb_flow_set_listener_state");
    }
    /// the same from d_tension and d_x on the flow's device, after the caller's work on `stream`
    void set_listener_state_device(const std::vector<skb_fiber_params> &params, double dt, double eta,
                                   const double *d_tension, const double *d_x, const std::vector<int32_t> &body_kind,
                                   const M &body_radii, bool periphery_interaction, void *stream = nullptr) {
        check(skb_flow_set_listener_state_device(st_->fl, params.data(), dt, eta, d_tension, d_x, body_kind.data(),
                                                 body_radii.data(), periphery_interaction ? 1 : 0, stream),
              "skb_flow_set_listener_state_device");
    }
    /// System::velocity_at_targets on the frame, the body-interior replacement included
    M listener_velocity(const M &r_trg) const {
        M vel = M::Zero(3, r_trg.cols());
        check(skb_flow_listener_velocity(st_->fl, r_trg.data(), r_trg.cols(), vel.data()), "skb_flow_listener_velocity");
        return vel;
    }
    /// StreamLine / VortexLine::compute of every seed (3 x n) at once: x and val are 3 x m, time m, per line
    struct Line {
        M x, val;
        std::vector<double> time;
        int32_t status[2];
    };
    std::vector<Line> listener_lines(int kind, const M &x0, const skb_line_request &req) const {
        const int n = (int)x0.cols();
        const long row = 2L * req.max_points - 1;
        std::vector<double> x(3 * n * std::max(row, 1L)), t(n * std::max(row, 1L)), val(x.size());
        std::vector<int32_t> n_points(n), status(2 * n);
        check(skb_flow_listener_lines(st_->fl, kind, x0.data(), n, &req, x.data(), t.data(), val.data(),
                                      n_points.data(), status.data()),
              "skb_flow_listener_lines");
        std::vector<Line> out(n);
        for (int i = 0; i < n; ++i) {
            const int m = n_points[i];
            out[i].x = M::Zero(3, m);
            out[i].val = M::Zero(3, m);
            std::copy_n(x.data() + 3 * row * i, 3 * m, out[i].x.data());
            std::copy_n(val.data() + 3 * row * i, 3 * m, out[i].val.data());
            out[i].time.assign(t.begin() + row * i, t.begin() + row * i + m);
            out[i].status[0] = status[2 * i];
            out[i].status[1] = status[2 * i + 1];
        }
        return out;
    }

    // ---- per-fiber dense operators on the device (SURVEY.md §8f N2) ----
    /// FiberFiniteDifference::matrices_.at(n_nodes): D_1_0 (n x n), P_downsample_bc ((4n-14) x 4n)  ffd.cpp:537-555
    void set_fiber_class(int n_nodes, const M &D_1_0, const M &P_downsample_bc) {
        check(skb_flow_set_fiber_class(st_->fl, n_nodes, D_1_0.data(), P_downsample_bc.data()),
              "skb_flow_set_fiber_class");
    }
    /// Once per timestep after set_fibers: A[f] / force_operator[f] point at fib.A_.data() / fib.force_operator_.data()
    /// (column-major 4n x 4n / 3n x 4n); xs = 3 x N_f tangents; length_prev / plus_bc_velocity per fiber.
    void set_fiber_operators(const std::vector<const double *> &A, const std::vector<const double *> &force_operator,
                             const M &xs, const std::vector<double> &length_prev,
                             const std::vector<int> &plus_bc_velocity) {
        const size_t nf = st_->n_nodes.size();
        if (A.size() != nf || force_operator.size() != nf || length_prev.size() != nf || plus_bc_velocity.size() != nf)
            throw std::runtime_error("skelly_b200: set_fiber_operators needs one entry per fiber of set_fibers");
        size_t na = 0, nfo = 0;
        for (int n : st_->n_nodes) {
            na += (size_t)16 * n * n;
            nfo += (size_t)12 * n * n;
        }
        std::vector<double> a(na), fo(nfo);
        size_t oa = 0, of = 0;
        for (size_t f = 0; f < nf; ++f) {
            const size_t n = (size_t)st_->n_nodes[f];
            std::copy(A[f], A[f] + 16 * n * n, a.begin() + oa);
            std::copy(force_operator[f], force_operator[f] + 12 * n * n, fo.begin() + of);
            oa += 16 * n * n;
            of += 12 * n * n;
        }
        check(skb_flow_set_fiber_operators(st_->fl, a.data(), fo.data(), xs.data(), length_prev.data(),
                                           plus_bc_velocity.data()),
              "skb_flow_set_fiber_operators");
    }
    /// A_inv[f] points at the column-major 4n x 4n inverse of fiber f's A_ (e.g. MatrixXd(fib.A_LU_.inverse()).data())
    void set_fiber_preconditioner(const std::vector<const double *> &A_inv) {
        const size_t nf = st_->n_nodes.size();
        if (A_inv.size() != nf)
            throw std::runtime_error("skelly_b200: set_fiber_preconditioner needs one entry per fiber of set_fibers");
        size_t na = 0;
        for (int n : st_->n_nodes)
            na += (size_t)16 * n * n;
        std::vector<double> a(na);
        size_t oa = 0;
        for (size_t f = 0; f < nf; ++f) {
            const size_t n = (size_t)st_->n_nodes[f];
            std::copy(A_inv[f], A_inv[f] + 16 * n * n, a.begin() + oa);
            oa += 16 * n * n;
        }
        check(skb_flow_set_fiber_preconditioner(st_->fl, a.data()), "skb_flow_set_fiber_preconditioner");
    }
    /// FiberFiniteDifference::matrices_.at(n_nodes): D_2_0, D_3_0, D_4_0 (n x n each, pre-transposed like D_1_0,
    /// ffd.cpp:537-540); build_fiber_operators needs them, and set_fiber_class, for every node count in use
    void set_fiber_class_derivatives(int n_nodes, const M &D_2_0, const M &D_3_0, const M &D_4_0) {
        check(skb_flow_set_fiber_class_derivatives(st_->fl, n_nodes, D_2_0.data(), D_3_0.data(), D_4_0.data()),
              "skb_flow_set_fiber_class_derivatives");
    }
    /// Once per timestep after set_fibers, instead of set_fiber_operators + set_fiber_preconditioner: A_,
    /// force_operator_, xs_ and A_^-1 of every fiber built on the device from the positions and lengths of set_fibers
    /// (update_derivatives, update_linear_operator, update_force_operator, apply_bc_rectangular's operator half,
    /// update_preconditioner); one skb_fiber_params per fiber
    void build_fiber_operators(const std::vector<skb_fiber_params> &params, double dt, double eta) {
        if (params.size() != st_->n_nodes.size())
            throw std::runtime_error("skelly_b200: build_fiber_operators needs one entry per fiber of set_fibers");
        check(skb_flow_build_fiber_operators(st_->fl, params.data(), dt, eta), "skb_flow_build_fiber_operators");
    }
    /// The fiber block of System::get_rhs (4 N_f) as System::prep_state_for_solver leaves it: fc.update_rhs(dt,
    /// v_on_fibers, motor + f_external), then fc.apply_bcs(dt, v_on_fibers, f_external), formed on the device.
    /// v_growth / force_scale per fiber (empty: zero growth / no motors); v_on_fibers / f_external 3 x N_f (size 0: the
    /// reference's empty matrix).  Needs set_fiber_class and set_fiber_class_derivatives, not the operators.
    M build_fiber_rhs(const std::vector<skb_fiber_params> &params, const std::vector<double> &v_growth,
                      const std::vector<double> &force_scale, const M &v_on_fibers, const M &f_external, double dt,
                      double eta) const {
        const size_t nfib = st_->n_nodes.size();
        if (params.size() != nfib || (!v_growth.empty() && v_growth.size() != nfib) ||
            (!force_scale.empty() && force_scale.size() != nfib))
            throw std::runtime_error("skelly_b200: build_fiber_rhs needs one entry per fiber of set_fibers");
        M rhs = M::Zero(4 * st_->n_fib, 1);
        check(skb_flow_build_fiber_rhs(st_->fl, params.data(), v_growth.empty() ? nullptr : v_growth.data(),
                                       force_scale.empty() ? nullptr : force_scale.data(),
                                       v_on_fibers.size() > 0 ? v_on_fibers.data() : nullptr,
                                       f_external.size() > 0 ? f_external.data() : nullptr, dt, eta, rhs.data()),
              "skb_flow_build_fiber_rhs");
        return rhs;
    }
    /// The resident operators back, in set_fiber_operators' layouts: A / A_inv the concatenated column-major 4n x 4n
    /// matrices, force_operator the 3n x 4n ones, xs 3 x N_f
    void get_fiber_operators(std::vector<double> &A, std::vector<double> &force_operator, M &xs,
                             std::vector<double> &A_inv) const {
        size_t na = 0;
        for (int n : st_->n_nodes)
            na += (size_t)16 * n * n;
        A.assign(na, 0.0);
        force_operator.assign(na / 4 * 3, 0.0);
        A_inv.assign(na, 0.0);
        xs = M::Zero(3, st_->n_fib);
        check(skb_flow_get_fiber_operators(st_->fl, A.data(), force_operator.data(), xs.data(), A_inv.data()),
              "skb_flow_get_fiber_operators");
    }
    /// FiberContainerFiniteDifference::apply_preconditioner (fcfd.cpp:331-339): y = A_^-1 x per fiber
    M apply_fiber_preconditioner(const M &x_fibers) const {
        M y = M::Zero(4 * st_->n_fib, 1);
        check(skb_flow_apply_fiber_preconditioner(st_->fl, x_fibers.data(), y.data()),
              "skb_flow_apply_fiber_preconditioner");
        return y;
    }
    /// FiberContainerFiniteDifference::apply_fiber_force (fcfd.cpp:272-287): x_fibers (4 N_f) -> 3 x N_f
    M apply_fiber_force(const M &x_fibers) const {
        M fw = M::Zero(3, st_->n_fib);
        check(skb_flow_apply_fiber_force(st_->fl, x_fibers.data(), fw.data()), "skb_flow_apply_fiber_force");
        return fw;
    }
    /// FiberContainerFiniteDifference::matvec (fcfd.cpp:216-232); v_fib_boundary 7 x n_fibers (size 0: none)
    M fiber_matvec(const M &x_fibers, const M &v_fibers, const M &v_fib_boundary) const {
        M res = M::Zero(4 * st_->n_fib, 1);
        check(skb_flow_fiber_matvec(st_->fl, x_fibers.data(), v_fibers.data(),
                                    v_fib_boundary.size() > 0 ? v_fib_boundary.data() : nullptr, res.data()),
              "skb_flow_fiber_matvec");
        return res;
    }
    /// System::apply_matvec (system.cpp:298-318) with fw and v_fibers kept on the device: returns res_fibers (4 N_f)
    /// and fills v_shell (3 x N_s) / v_bodies (3 x N_b) for shell.matvec / bc.matvec.
    M apply_matvec(const M &x_fibers, const M &shell_density, const M &body_densities, const M &forces_torques,
                   const M &fiber_link_conditions, double eta, M &v_shell, M &v_bodies) const {
        M res = M::Zero(4 * st_->n_fib, 1);
        v_shell = M::Zero(3, st_->n_shell);
        v_bodies = M::Zero(3, st_->n_body);
        check(skb_flow_apply_matvec(st_->fl, x_fibers.data(), shell_density.data(), body_densities.data(),
                                    forces_torques.data(),
                                    fiber_link_conditions.size() > 0 ? fiber_link_conditions.data() : nullptr, eta,
                                    res.data(), v_shell.data(), v_bodies.data()),
              "skb_flow_apply_matvec");
        return res;
    }
    /// The same with shell.matvec on the device: `dn` holds stresslet_plus_complementary_ (skelly_b200_dense.h);
    /// res_shell (3 N_s) = stresslet_plus_complementary_ * x_shell + v_shell  (system.cpp:319, periphery.cpp:38-47)
    M apply_matvec(skb_dense *dn, const M &x_fibers, const M &x_shell, const M &body_densities,
                   const M &forces_torques, const M &fiber_link_conditions, double eta, M &res_shell,
                   M &v_bodies) const {
        M res = M::Zero(4 * st_->n_fib, 1);
        res_shell = M::Zero(3 * st_->n_shell, 1);
        v_bodies = M::Zero(3, st_->n_body);
        check(skb_flow_apply_matvec_dense(st_->fl, dn, x_fibers.data(), x_shell.data(), body_densities.data(),
                                          forces_torques.data(),
                                          fiber_link_conditions.size() > 0 ? fiber_link_conditions.data() : nullptr,
                                          eta, res.data(), res_shell.data(), v_bodies.data()),
              "skb_flow_apply_matvec_dense");
        return res;
    }
    // ---- the whole solution vector [fibers | shell | bodies] with the bodies on the device (one GPU) ----
    /// Once per timestep after set_bodies, per body in the order of the solution vector: n_nodes, node_weights_ (N_b),
    /// ex_ / ey_ / ez_ (3 x N_b each, body_spherical.cpp:168-181) and A_inv = the column-major (3n+6)^2 inverses of A_,
    /// concatenated (empty: the system preconditioner refuses bodies)
    void set_body_operators(const std::vector<int> &n_nodes, const std::vector<double> &node_weights, const M &ex,
                            const M &ey, const M &ez, const std::vector<double> &A_inv) {
        check(skb_flow_set_body_operators(st_->fl, n_nodes.data(), (int)n_nodes.size(), node_weights.data(), ex.data(),
                                          ey.data(), ez.data(), A_inv.empty() ? nullptr : A_inv.data()),
              "skb_flow_set_body_operators");
    }
    /// Once per timestep after set_fibers / set_bodies, per fiber: body index (binding_site_.first, -1 = free), lab-frame
    /// nucleation site (3 x n_fibers), bending_rigidity_; an empty `body`: no fiber is bound
    void set_fiber_links(const std::vector<int> &body, const M &site, const std::vector<double> &bending_rigidity) {
        if (!body.empty() && (body.size() != st_->n_nodes.size() || bending_rigidity.size() != body.size()))
            throw std::runtime_error("skelly_b200: set_fiber_links needs one entry per fiber of set_fibers");
        check(skb_flow_set_fiber_links(st_->fl, body.empty() ? nullptr : body.data(), site.data(),
                                       bending_rigidity.data()),
              "skb_flow_set_fiber_links");
    }
    /// System::apply_matvec (system.cpp:269-324) on the whole solution vector; dn holds stresslet_plus_complementary_
    M apply_system_matvec(skb_dense *dn, const M &x, double eta) const {
        M res = M::Zero(x.size(), 1);
        check(skb_flow_apply_system_matvec(st_->fl, dn, x.data(), eta, res.data()), "skb_flow_apply_system_matvec");
        return res;
    }
    /// System::apply_preconditioner (system.cpp:248-262) on the whole solution vector; dn holds M_inv_
    M apply_system_preconditioner(skb_dense *dn, const M &x) const {
        M y = M::Zero(x.size(), 1);
        check(skb_flow_apply_system_preconditioner(st_->fl, dn, x.data(), y.data()),
              "skb_flow_apply_system_preconditioner");
        return y;
    }
    // ---- switches of the matvec (all optional; defaults are the fast paths with the reference's semantics) ----
    /// fibers <-> periphery pairs in one geometry pass: -1 auto (default), 0 never, 1 whenever applicable
    void set_cross(int mode) { check(skb_flow_set_cross(st_->fl, mode), "skb_flow_set_cross"); }
    /// the pair kernels skip intra-fiber pairs instead of the reference's compute-then-subtract (fcfd.cpp:203-210)
    void set_self_exclusion(bool fused) {
        check(skb_flow_set_self_exclusion(st_->fl, fused ? 1 : 0), "skb_flow_set_self_exclusion");
    }
    /// Periphery::matvec's dense operator beside the pair kernels on a side stream (default) or after them
    void set_overlap(bool on) { check(skb_flow_set_overlap(st_->fl, on ? 1 : 0), "skb_flow_set_overlap"); }
    skb_flow *handle() const { return st_->fl; }

  private:
    struct State { // copies of the engine share the device state and the geometry sizes, like the evaluators
        skb_flow *fl = nullptr;
        long n_fib = 0, n_shell = 0, n_body = 0;
        std::vector<int> n_nodes;
        ~State() { skb_flow_destroy(fl); }
    };
    std::shared_ptr<State> st_;
};

using FlowEngine = FlowEngineT<Matrix>;

} // namespace skelly_b200

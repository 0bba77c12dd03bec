"""Restatement of the listener's frame of a solution in numpy: what the reference's listener does with a trajectory frame
(trajectory_reader.cpp:150-249) before System::velocity_at_targets evaluates it (system.cpp:330-384), in the order of
skb_flow_set_listener_state (include/skelly_b200_flow.h):

  1. sol_fibers per fiber = [x; y; z; T] from the frame's positions x_ and tension_ (trajectory_reader.cpp:238-246), not
     from the fiber block of the solution;
  2. fc.update_cache_variables(dt, eta) at those positions (:248): force_operator_ and xs_ (oracle.fiber_fd);
  3. f_on_fibers = fc.apply_fiber_force(sol_fibers), + fc.periphery_force(shell, fp) only with
     periphery_interaction_flag (system.cpp:339-341); no motor force;
  4. body_link_conditions of calculate_link_conditions(sol_fibers, sol_bodies) (:349-350; system_reference.
     link_conditions); calculate_external_forces_torques is computed at :352 and not passed to bc_.flow (:356);
  5. the shell density is the shell block, the body densities the first 3 n_b entries of each body's block;
  6. each body's [U; omega] the last six entries of its block (SphericalBody::step, body_spherical.cpp:16-17).

DEFECTS are planted departures from that reading, for the tests that show the restatement tells them apart."""
import numpy as np

import periphery_reference as pr
import system_reference as sr
from oracle.fiber_fd import FiberOperators, compute_matrices

DEFECTS = ("gmres_fibers", "motor_force", "external_ft", "uw_offset", "repulsion_flag_off")


def _operators(fib, params, dt, eta):
    """FiberOperators of every fiber at its positions; params: the seven per-fiber arrays of skb_fiber_params"""
    lp, E, radius, penalty, beta, clamped, hinged = (np.broadcast_to(np.asarray(v), (len(fib["n_nodes"]),))
                                                   for v in params)
    out, off = [], 0
    for f, n in enumerate(fib["n_nodes"]):
        out.append(FiberOperators(fib["pos"][off:off + n], fib["lengths"][f], bending_rigidity=E[f], radius=radius[f],
                                  eta=eta, dt=dt, length_prev=lp[f], minus_clamped=bool(clamped[f]),
                                  plus_pinned=bool(hinged[f]), penalty_param=penalty[f], beta_tstep=beta[f]))
        off += n
    return out


def frame(fib, n_shell, bodies, links, params, dt, eta, x, tension, shape=None, shape_minus_clamped=None,
          periphery_interaction=False, external_ft=None, force_scale=None, defect=None):
    """The strengths of the frame: dict(fib_forces (N_f, 3), shell_density (N_s, 3), body_densities (N_b, 3),
    body_ft (n_bodies, 6), body_uw (n_bodies, 6)).

    fib: dict(pos (N_f, 3), n_nodes, lengths); bodies: dict(n_nodes, centers); links: dict(body, site, rigidity) per
    fiber (body -1 free) or None; x: the step's whole solution vector; tension (N_f,); shape: a periphery_reference
    shape dict with shape_minus_clamped its per-fiber flags.  external_ft (n_bodies, 6) and force_scale (per fiber) are
    what the reference has at hand and leaves out; the defects "external_ft" and "motor_force" put them in."""
    assert defect is None or defect in DEFECTS, defect
    n_nodes = [int(n) for n in fib["n_nodes"]]
    nf = int(sum(n_nodes))
    x = np.asarray(x, dtype=np.float64)
    x_f, x_s, x_b = sr.split(x, nf, n_shell)
    ops = _operators(fib, params, dt, eta)
    off = np.concatenate([[0], np.cumsum(n_nodes)]).astype(int)
    sol_fibers, ff = [], np.zeros((nf, 3))
    for f, (n, op) in enumerate(zip(n_nodes, ops)):
        a = off[f]
        if defect == "gmres_fibers":
            s = x_f[4 * a:4 * a + 4 * n]
        else:
            s = np.concatenate([fib["pos"][a:a + n].T.reshape(-1), np.asarray(tension[a:a + n], dtype=np.float64)])
        sol_fibers.append(s)
        ff[a:a + n] = (op.force_operator @ s).reshape(3, n).T                  # apply_fiber_force, fcfd.cpp:272-287
        if defect == "motor_force":                                            # generate_constant_force: force_scale xs
            ff[a:a + n] += np.asarray(force_scale)[f] * op.xs
        if periphery_interaction or defect == "repulsion_flag_off":
            clamped = bool(shape_minus_clamped[f]) if shape_minus_clamped is not None else False
            ff[a:a + n] += pr.fiber_interaction(shape, fib["pos"][a:a + n], clamped)
    sol_fibers = np.concatenate(sol_fibers) if sol_fibers else np.zeros(0)
    nb = len(bodies["n_nodes"])
    ft = np.zeros((nb, 6))
    if nb and links is not None and nf:
        lops = dict(xs=np.concatenate([op.xs for op in ops]), length_prev=[op.length_prev for op in ops],
                    D_2_0={n: compute_matrices(n)["D_2_0"] for n in n_nodes},
                    D_3_0={n: compute_matrices(n)["D_3_0"] for n in n_nodes})
        _, ft = sr.link_conditions(fib, lops, links, bodies, sol_fibers, x_b)
    if defect == "external_ft":
        ft = ft + np.asarray(external_ft)
    node_off, sol_off = sr._body_offsets(bodies["n_nodes"])
    dens, uw = np.zeros((int(node_off[-1]), 3)), np.zeros((nb, 6))
    for b, n in enumerate(bodies["n_nodes"]):
        s = int(sol_off[b])
        dens[node_off[b]:node_off[b + 1]] = x_b[s:s + 3 * n].reshape(n, 3)
        u0 = s if defect == "uw_offset" else s + 3 * n
        uw[b] = x_b[u0:u0 + 6]
    return dict(fib_forces=ff, shell_density=x_s.reshape(-1, 3), body_densities=dens, body_ft=ft, body_uw=uw)


def gate(a, b):
    """the largest relative difference of any block (max-norm over the block, relative to b's): the 1e-12 gate"""
    worst = 0.0
    for k in b:
        scale = np.abs(b[k]).max() if b[k].size else 0.0
        d = np.abs(a[k] - b[k]).max() if b[k].size else 0.0
        worst = max(worst, d / scale if scale > 0 else (0.0 if d == 0 else np.inf))
    return worst

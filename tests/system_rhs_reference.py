"""CPU restatement of the right-hand side of the mobility system -- TEST INFRASTRUCTURE ONLY.

System::prep_state_for_solver (system.cpp:398-458) as Solver::set_RHS copies it (solver_hydro.cpp:51-61), on the
solution layout of system_reference.split: [fibers (4 per node) | shell (3 per node) | bodies (3 n_b + 6 each)].
Citations are `file:line` in the SkellySim tree.  The six steps:

  1. v_all = fc.flow(r_all, f_ext, eta) at [fibers | periphery | bodies], self term subtracted (:425); motor forces
     are not in this flow (:424)
  2. v_all += bc.flow(r_all, 0, F_T, eta) when any external F_T is nonzero: centre Stokeslet + rotlet (:431-443)
  3. v_all += psc.flow(r_all, eta, t) + bs.flow(r_all, eta) (:445-446)
  4. body b: [-v of its nodes ; 0 0 0 0 0 0] (body_spherical.cpp:134-138)
  5. fibers: update_rhs(dt, v_fibers, motor + f_ext), apply_bcs(dt, v_fibers, f_ext) (:451-453) =
     fiber_rhs_reference.fiber_rhs per fiber
  6. shell: -v_shell (periphery.cpp:86)

Dicts: fib = dict(pos, n_nodes, lengths); shell = dict(pos, normals); bodies = dict(pos, normals, centers, n_nodes);
fparams = per-fiber FiberOperators keywords (length_prev, bending_rigidity, radius, penalty_param, beta_tstep,
minus_clamped, plus_pinned); points = (positions, forces, torques) or None; background = (components, scale, uniform)
or None."""
import numpy as np

import oracle as orc
from fiber_rhs_reference import fiber_rhs
from oracle import fiber_fd

# defects a test of the RHS must catch: the motor force in the flow of step 1; the self term not subtracted; each F_T
# counted twice (once per member of a two-member group); the body rows +v; the six rows not zero (F_T in them); the
# point sources evaluated at the rows of the next node
RHS_DEFECTS = ("motor_in_flow", "no_self", "ft_twice", "body_sign", "six_nonzero", "points_wrong_rows")


def fiber_operators(fib, fparams, eta, dt, **kw):
    """oracle FiberOperators of every fiber (kw: dtype / absolute, as FiberOperators takes them)"""
    out, off = [], 0
    for f, (n, L) in enumerate(zip(fib["n_nodes"], fib["lengths"])):
        n = int(n)
        out.append(fiber_fd.FiberOperators(np.asarray(fib["pos"][off:off + n]), float(L), eta=eta, dt=dt,
                                           **fparams[f], **kw))
        off += n
    return out


def flow(fib, shell, bodies, eta, f_ext=None, ft=None, points=None, background=None, fos=None, force_scale=None,
         defect=None):
    """v_all of steps 1-3, (N_f + N_s + N_b, 3)"""
    r_f, r_s, r_b = (np.asarray(d["pos"], dtype=np.float64).reshape(-1, 3) for d in (fib, shell, bodies))
    nf = r_f.shape[0]
    r_all = np.concatenate([r_f, r_s, r_b])
    f = np.zeros((nf, 3)) if f_ext is None else np.array(f_ext, dtype=np.float64).reshape(nf, 3)
    if defect == "motor_in_flow" and force_scale is not None:
        f = f + np.concatenate([s * fo.xs for s, fo in zip(force_scale, fos)])
    v = orc.fiber_flow(r_all, r_f, fib["n_nodes"], fib["lengths"], f, eta, subtract_self=defect != "no_self")
    if ft is not None and np.any(ft):
        k = 2.0 if defect == "ft_twice" else 1.0
        ft = np.asarray(ft, dtype=np.float64).reshape(-1, 6)
        v += orc.body_flow(r_all, r_b, bodies["normals"], np.zeros_like(r_b), bodies["centers"], k * ft[:, :3],
                           k * ft[:, 3:], eta)
    if points is not None:
        pos, pf, pt = points
        r_eval = np.roll(r_all, 1, axis=0) if defect == "points_wrong_rows" else r_all
        v += orc.oseen_contract(pos, r_eval, pf, eta) + orc.rotlet(pos, r_eval, pt, eta)
    if background is not None:
        comp, scale, uni = background
        v += np.asarray(uni)[None, :] + r_all[:, list(comp)] * np.asarray(scale)[None, :]
    return v


def system_rhs(fib, shell, bodies, fparams, eta, dt, f_ext=None, ft=None, points=None, background=None,
               v_growth=None, force_scale=None, defect=None):
    """The whole RHS vector; v_growth / force_scale per fiber or None.  Returns (rhs, v_all)."""
    assert defect is None or defect in RHS_DEFECTS, defect
    fos = fiber_operators(fib, fparams, eta, dt)
    v = flow(fib, shell, bodies, eta, f_ext, ft, points, background, fos, force_scale, defect)
    nf, ns = int(np.sum(fib["n_nodes"], dtype=np.int64)), np.asarray(shell["pos"]).reshape(-1, 3).shape[0]
    out, off = [], 0
    for f, fo in enumerate(fos):
        n = fo.n
        out.append(fiber_rhs(fo, v=v[off:off + n], f_external=None if f_ext is None else np.asarray(f_ext)[off:off + n],
                             force_scale=None if force_scale is None else force_scale[f],
                             v_growth=0.0 if v_growth is None else v_growth[f]))
        off += n
    out.append(-v[nf:nf + ns].reshape(-1))
    sign = 1.0 if defect == "body_sign" else -1.0
    node = nf + ns
    for b, n in enumerate(bodies["n_nodes"]):
        out.append(sign * v[node:node + n].reshape(-1))
        six = np.zeros(6)
        if defect == "six_nonzero" and ft is not None:
            six = np.asarray(ft, dtype=np.float64).reshape(-1, 6)[b]
        out.append(six)
        node += n
    return np.concatenate(out) if out else np.zeros(0), v

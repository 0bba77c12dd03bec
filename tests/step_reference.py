"""numpy restatement of System::step's pieces and System::run's acceptance (system.cpp:482-568), for the CPU tests
(tests/test_step_cpu.py) and the GPU tests of skb_flow_step (tests/test_gpu_step.py).

  fiber_step        FiberContainerFiniteDifference::step (fcfd.cpp:292-302): [x(n); y(n); z(n); T(n)] per fiber
  repin             ::repin_to_bodies (fcfd.cpp:308-316): delta = site - x_0, then x_i + delta
  body_step         SphericalBody::step (body_spherical.cpp:13-35): literal=True the reference's rule, else the rule
                    skb_flow_step takes (always translate, normalise q)
  fiber_error       ::fiber_error_local (fcfd.cpp:79-89), in float64 or np.longdouble, with an error scale S
  run_reference     System::run's acceptance, time advanced by the grown dt as the reference does (literal) or by the
                    dt the step used"""
import math

import numpy as np


def fiber_step(x_fib, n_nodes):
    """per fiber (positions (n, 3), tension (n,)) of the solution's fiber block"""
    out, off = [], 0
    for n in n_nodes:
        blk = x_fib[off:off + 4 * n]
        out.append((blk[:3 * n].reshape(3, n).T.copy(), blk[3 * n:].copy()))
        off += 4 * n
    return out


def repin(pos, site, from_last=False):
    """positions moved so that node 0 lies at site (from_last: the planted defect of measuring from the last node)"""
    delta = site - (pos[-1] if from_last else pos[0])
    return pos + delta


def quat_mul(a, b):
    """Eigen's quaternion product a * b, (w, x, y, z)"""
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
                     a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3],
                     a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]])


def rotation(q):
    """Eigen's toRotationMatrix of a unit quaternion (w, x, y, z), in its operation order"""
    w, x, y, z = q
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return np.array([[1.0 - (tyy + tzz), txy - twz, txz + twy],
                     [txy + twz, 1.0 - (txx + tzz), tyz - twx],
                     [txz - twy, tyz + twx, 1.0 - (txx + tyy)]])


def body_step(c, q, U, w, dt, literal=False, right=False):
    """(c_new, q_new) of one body from its rows U, w.  literal: the reference's rule -- the body moves only when
    |phi| != 0 (place() is called only then) and q_new is not normalised.  right: the planted defect q * q_phi"""
    c, q = np.asarray(c, float), np.asarray(q, float)
    phi = [float(w[k]) * dt for k in range(3)]
    pn = math.sqrt(phi[0] * phi[0] + phi[1] * phi[1] + phi[2] * phi[2])
    c_new = np.array([float(c[k]) + float(U[k]) * dt for k in range(3)])
    if pn == 0.0:
        return (c.copy() if literal else c_new), q.copy()
    sh = math.sin(0.5 * pn)
    qp = np.array([math.cos(0.5 * pn), sh * phi[0] / pn, sh * phi[1] / pn, sh * phi[2] / pn])
    r = quat_mul(q, qp) if right else quat_mul(qp, q)
    if literal:
        return c_new, r
    return c_new, r / np.sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3])


def site(c, q, s_ref, rotate=True):
    """get_nucleation_site: c + R(q) s_ref, R applied in the device's order (rotate=False: the planted defect of sites
    left in the body frame)"""
    if not rotate:
        return np.asarray(c) + np.asarray(s_ref)
    R = rotation(q)
    return np.array([c[k] + (R[k, 0] * s_ref[0] + R[k, 1] * s_ref[1] + R[k, 2] * s_ref[2]) for k in range(3)])


def fiber_error(pos, length, D, dtype=np.float64, scale=2.0):
    """(per node | ||xs_i|| - 1 |, per node error scale S_i) with xs = (scale / length) x D_1_0 evaluated in dtype.
    S_i = (2/L) ||(sum_j |x_kj| |D_ji|)_k|| + ||xs_i|| + 1 bounds what rounding of the sums, the norm and the
    difference can move the error by, in units of u"""
    x = np.asarray(pos, dtype=dtype).T
    Dd = np.asarray(D, dtype=dtype)
    xs = (dtype(scale) / dtype(length)) * (x @ Dd)
    nrm = np.sqrt((xs * xs).sum(axis=0))
    S = (2.0 / float(length)) * np.linalg.norm(np.abs(np.asarray(pos, float)).T @ np.abs(np.asarray(D, float)), axis=0)
    return np.abs(nrm - dtype(1)), S + np.asarray(nrm, float) + 1.0


def run_reference(outcomes, dt, t_final, dt_min, dt_max, beta_up, beta_down, tol, adaptive=True, literal=False):
    """System::run's decisions over scripted (converged, fiber_error, collided) outcomes: a list of (time after, dt used,
    accepted) per step; literal: time advanced by the dt after its update, as system.cpp:554-557 does"""
    time, out, k = 0.0, [], 0
    while time < t_final:
        converged, err, collided = outcomes[k]
        k += 1
        dt_new, accept = dt, False
        if adaptive:
            if converged and err <= tol:
                accept = True
                if err <= 0.9 * tol:
                    dt_new = min(dt_max, dt * beta_up)
            else:
                dt_new = dt * beta_down
            if converged and collided:
                dt_new, accept = dt * 0.5, False
            if dt_new < dt_min:
                raise RuntimeError("Timestep smaller than dt_min")
        used = dt
        if adaptive and literal:
            dt = dt_new
        if not adaptive or accept:
            time += dt if literal else used
        out.append((time, used, accept))
        dt = dt_new
    return out

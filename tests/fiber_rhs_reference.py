"""CPU restatement of the fiber block of the RHS -- TEST INFRASTRUCTURE ONLY.

fiber_rhs(fo, ...) gives RHS_ of the fiber whose operators oracle/fiber_fd.py::FiberOperators `fo` holds, as
System::prep_state_for_solver leaves it (system.cpp:416-453): update_RHS(dt, v, f_external + force_scale xs_)
(fiber_finite_difference.cpp:198-274), then the RHS half of apply_bc_rectangular(dt, v, f_external) (:358-504).
Citations are `file:line` in the SkellySim tree.  It follows FiberOperators' conventions: the arithmetic is fo's dtype
(np.longdouble evaluates exactly the function of the float64 inputs that a float64 evaluation rounds), and an fo built
with absolute=True gives the error scale S (every input by its absolute value, every subtraction an addition)."""
import numpy as np

from oracle.fiber_fd import BC_VELOCITY

# defects a test of the kernel must catch: D_1 of update_RHS scaled by length_prev_, f_tot in the boundary entries, the
# s_dot term dropped, the (c_0 - c_1) xss . f term dropped, the minus / plus boundary-condition branches swapped
RHS_DEFECTS = ("d1_length_prev", "ftot_in_bc", "no_sdot", "no_xss_f", "swap_bc")


def fiber_rhs(fo, v=None, f_external=None, force_scale=None, v_growth=0.0, defect=None):
    """(4n,) RHS_ of one fiber.  v, f_external: (n, 3) or None (the reference's empty matrix); force_scale None: no
    motor force (generate_constant_force, fcfd.cpp:160-169); defect: one of RHS_DEFECTS or None."""
    assert defect is None or defect in RHS_DEFECTS, defect
    n, m, sg, f = fo.n, fo._m, fo.sg, fo.dtype
    absolute = sg > 0
    mag = (lambda b: np.abs(b)) if absolute else (lambda b: b)
    cv = lambda a: None if a is None else mag(np.asarray(a, dtype=np.float64).astype(f).reshape(n, 3))
    sc = lambda s: mag(f(np.float64(s)))
    v, fe = cv(v), cv(f_external)
    x, xs, xss, dt, c0, c1 = fo.x, fo.xs, fo.xss, fo.dt, fo.c_0, fo.c_1
    # f_tot = motor + external (system.cpp:450)
    motor = None if force_scale is None else sc(force_scale) * xs
    ft = fe if motor is None else (motor if fe is None else motor + fe)

    # update_RHS (ffd.cpp:198-274)
    D_1 = m["D_1_0"] * (2.0 / (fo.length_prev if defect == "d1_length_prev" else fo.length))               # :201
    alpha = fo.mats["alpha"].astype(f)
    s_dot = (1.0 + mag(alpha)) * (0.5 * sc(v_growth))                                                  # :211-212
    if defect == "no_sdot":
        s_dot = s_dot * 0
    R = np.zeros(4 * n, dtype=f)
    for a in range(3):                                                                                 # :218-220
        R[a * n:(a + 1) * n] = x[:, a] / dt + s_dot * xs[:, a]
    R[3 * n:] = sg * fo.penalty * np.ones(n, dtype=f)                                                  # :221
    if v is not None:                                                                                  # :223-232
        for a in range(3):
            R[a * n:(a + 1) * n] += v[:, a]
        R[3 * n:] += xs[:, 0] * (v[:, 0] @ D_1) + xs[:, 1] * (v[:, 1] @ D_1) + xs[:, 2] * (v[:, 2] @ D_1)
    if ft is not None:                                                                                 # :233-273
        fs = [ft[:, b] @ D_1 for b in range(3)]
        for a in range(3):
            t = 0
            for cc, s in ((c0, 1.0), (c1, sg)):
                for b in range(3):
                    t = t + cc * (((1.0 if a == b else 0.0) + s * xs[:, a] * xs[:, b]) * ft[:, b])
            R[a * n:(a + 1) * n] += t
        R[3 * n:] += 2 * c0 * (xs[:, 0] * fs[0] + xs[:, 1] * fs[1] + xs[:, 2] * fs[2])
        if defect != "no_xss_f":
            R[3 * n:] += (c0 + sg * c1) * (xss[:, 0] * ft[:, 0] + xss[:, 1] * ft[:, 1] + xss[:, 2] * ft[:, 2])

    # apply_bc_rectangular, RHS half (ffd.cpp:358-504): the boundary entries see f_external only
    out = np.zeros(4 * n, dtype=f)
    out[:4 * n - 14] = m["P_downsample_bc"] @ R                                                      # :359
    fb = ft if defect == "ftot_in_bc" else fe
    minus_vel, plus_vel = fo.bc_minus[0] == BC_VELOCITY, fo.bc_plus[0] == BC_VELOCITY
    if defect == "swap_bc":
        minus_vel, plus_vel = plus_vel, minus_vel
    B = np.zeros(14, dtype=f)
    for base, node, vel in ((0, 0, minus_vel), (7, n - 1, plus_vel)):
        if vel:                                                                    # Velocity :377-383, 457-463
            B[base:base + 3] = x[node] / dt
            if v is not None:
                B[base + 3] += sg * (xs[node] @ v[node])
            if fb is not None:
                B[base + 3] += sg * (2 * c0 * (xs[node] @ fb[node]))
        else:                                                                      # Force :399-404, 481-486
            vec = fb[node] if fb is not None else np.zeros(3, dtype=f)
            B[base:base + 3] = vec
            B[base + 3] = vec @ xs[node]
    if minus_vel:                                                                  # AngularVelocity :422-423
        B[4:7] = xs[0] / dt                                                        # (Torque: zero, :432-433, 502-504)
    out[4 * n - 14:] = B
    return out

"""Restatement of the listener's streamlines and vortex lines (StreamLine::compute / VortexLine::compute,
streamline.cpp) for any velocity callable -- TEST INFRASTRUCTURE ONLY.

The reference integrates with boost.odeint: integrate_adaptive over controlled_runge_kutta<runge_kutta_cash_karp54>,
with the default error checker (a_x = a_dxdt = 1), the default step adjuster (no max dt) and failed_step_checker's
limit of 500 tries.  boost is not part of this project's build or tests: the formulas here are restated from odeint's
source (integrate_adaptive, controlled_runge_kutta::try_step, default_error_checker, default_step_adjuster,
failed_step_checker), not compiled against it.

    while less_with_sign(t, T, dt):
        obs(x, t)                       # appends (x, t); ends the line (point kept) when |velocity(x)| > 1e3
        if less_with_sign(T, t + dt, dt): dt = T - t
        repeat try_step until success   # 500 consecutive failures end the line
    obs(x, t)

velocity(points) takes an (m, 3) array and returns the (m, 3) velocities there.
"""
import numpy as np

DBL_EPSILON = np.finfo(np.float64).eps
VORTEX_EPS = 1e-7   # get_vorticity_at_point (streamline.cpp:16-35)
SINGULAR_SPEED = 1e3
MAX_FAILS = 500
REACHED, SINGULAR, FAILED, CAPPED = 0, 1, 2, 3

# Cash-Karp 5(4): a_ij, the 5th-order weights b and b - b* (the 4th-order weights) of the error estimate
A = [[],
     [1 / 5],
     [3 / 40, 9 / 40],
     [3 / 10, -9 / 10, 6 / 5],
     [-11 / 54, 5 / 2, -70 / 27, 35 / 27],
     [1631 / 55296, 175 / 512, 575 / 13824, 44275 / 110592, 253 / 4096]]
B = [37 / 378, 0.0, 250 / 621, 125 / 594, 0.0, 512 / 1771]
B_STAR = [2825 / 27648, 0.0, 18575 / 48384, 13525 / 55296, 277 / 14336, 1 / 4]
DB = [b - bs for b, bs in zip(B, B_STAR)]


def less_with_sign(t1, t2, dt):
    """odeint's less_with_sign: t1 < t2 in the direction of dt, by more than DBL_EPSILON."""
    return t2 - t1 > DBL_EPSILON if dt > 0 else t1 - t2 > DBL_EPSILON


def vorticity(velocity, x):
    """get_vorticity_at_point: the curl from the six points x +- 1e-7 e_j, combined as streamline.cpp does."""
    p = np.repeat(np.asarray(x, dtype=np.float64)[None, :], 6, axis=0)
    for j in range(6):
        p[j, j // 2] = p[j, j // 2] - VORTEX_EPS if j % 2 else p[j, j // 2] + VORTEX_EPS
    v = velocity(p)  # v(c, j) of the reference is v[j, c]
    w = np.array([(v[2, 2] - v[3, 2]) - (v[4, 1] - v[5, 1]),
                  (v[4, 0] - v[5, 0]) - (v[0, 2] - v[1, 2]),
                  (v[0, 1] - v[1, 1]) - (v[2, 0] - v[3, 0])])
    return 0.5 * w / VORTEX_EPS


def cash_karp_step(deriv, x, dt, abs_err, rel_err, k1=None):
    """One runge_kutta_cash_karp54 step with its error estimate and default_error_checker's error:
    (x_new, err, k1)."""
    k = [deriv(x) if k1 is None else k1]
    for s in range(1, 6):
        xs = x.copy()
        for j in range(s):
            xs = xs + (dt * A[s][j]) * k[j]
        k.append(deriv(xs))
    x_new, x_err = x.copy(), np.zeros(3)
    for j in range(6):
        x_new = x_new + (dt * B[j]) * k[j]
        x_err = x_err + (dt * DB[j]) * k[j]
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.abs(x_err) / (abs_err + rel_err * (np.abs(x) + abs(dt) * np.abs(k[0])))
    err = 0.0
    for v in e:  # norm_inf with std::max: a NaN never replaces the running maximum
        err = v if err < v else err
    return x_new, float(err), k[0]


def decrease_step(dt, err):
    """default_step_adjuster::decrease_step, error order 4."""
    f = 0.9 * err ** (-1.0 / 3.0)
    return dt * (0.2 if f < 0.2 else f)


def increase_step(dt, err):
    """default_step_adjuster::increase_step, stepper order 5."""
    if err < 0.5:
        err = err if 5.0 ** -5 < err else 5.0 ** -5
        dt *= 0.9 * err ** (-1.0 / 5.0)
    return dt


def integrate(deriv, velocity, x0, t_final, dt0, abs_err, rel_err, max_points=None, trace=None):
    """integrate_adaptive from t = 0 to t_final (negative for the back run) starting with dt0 (of t_final's sign).
    deriv(x) is the integrand at one point, velocity(x) the observer's velocity there.  Returns (points, times,
    vals, status); vals holds deriv at every point.  trace, a list, receives (t, dt, err, accepted) of every try."""
    x, t, dt = np.array(x0, dtype=np.float64), 0.0, float(dt0)
    T = float(t_final)
    pts, ts, vals = [], [], []

    def observe():
        k1 = deriv(x)
        pts.append(x.copy())
        ts.append(t)
        vals.append(k1)
        return k1, np.linalg.norm(velocity(x)) > SINGULAR_SPEED

    while less_with_sign(t, T, dt):
        k1, singular = observe()
        if singular:
            return np.array(pts), np.array(ts), np.array(vals), SINGULAR
        if max_points is not None and len(pts) >= max_points:
            return np.array(pts), np.array(ts), np.array(vals), CAPPED
        if less_with_sign(T, t + dt, dt):
            dt = T - t
        fails = 0
        while True:
            x_new, err, _ = cash_karp_step(deriv, x, dt, abs_err, rel_err, k1)
            if trace is not None:
                trace.append((t, dt, err, not err > 1.0))
            if err > 1.0:
                dt = decrease_step(dt, err)
                fails += 1
                if fails >= MAX_FAILS:
                    return np.array(pts), np.array(ts), np.array(vals), FAILED
                continue
            t += dt
            dt = increase_step(dt, err)
            x = x_new
            break
    _, singular = observe()
    return np.array(pts), np.array(ts), np.array(vals), SINGULAR if singular else REACHED


def join_back_and_forward(back, forward):
    """streamline.cpp's join: the back points reversed without their first (the seed), then the forward points."""
    return np.concatenate([back[:0:-1], forward]) if len(back) else forward


def lines(velocity, x0, kind=0, dt_init=0.1, t_final=1.0, abs_err=1e-10, rel_err=1e-6, back_integrate=True,
          max_points=None):
    """StreamLine::compute (kind 0) or VortexLine::compute (kind 1) of every seed in x0 (n, 3): a list of
    {"x", "time", "val", "status": (back, forward)} as skellysim_b200.Flow.streamlines returns them."""
    vel1 = lambda x: velocity(np.asarray(x, dtype=np.float64)[None, :])[0]  # noqa: E731
    deriv = vel1 if kind == 0 else (lambda x: vorticity(velocity, x))
    out = []
    for s in np.asarray(x0, dtype=np.float64).reshape(-1, 3):
        fx, ft, fv, fs = integrate(deriv, vel1, s, t_final, dt_init, abs_err, rel_err, max_points)
        if back_integrate:
            bx, bt, bv, bs = integrate(deriv, vel1, s, -t_final, -dt_init, abs_err, rel_err, max_points)
            fx, ft, fv = join_back_and_forward(bx, fx), join_back_and_forward(bt, ft), join_back_and_forward(bv, fv)
        else:
            bs = REACHED
        out.append({"x": fx, "time": ft, "val": fv, "status": (bs, fs)})
    return out

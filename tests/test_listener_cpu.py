"""CPU tests of tests/streamline_reference.py, the restatement of the listener's Cash-Karp streamline and vortex-line
integration (streamline.cpp over boost.odeint) that the device lines are checked against."""
import numpy as np
import pytest

import streamline_reference as sl


def rotation(points):
    # rigid rotation about z at unit rate: v = e_z x r
    p = np.asarray(points, dtype=np.float64)
    return np.stack([-p[:, 1], p[:, 0], np.zeros(len(p))], axis=1)


def shear(points, rate=0.7):
    p = np.asarray(points, dtype=np.float64)
    return np.stack([rate * p[:, 1], np.zeros(len(p)), np.zeros(len(p))], axis=1)


def constant(points):
    return np.tile([0.3, -0.2, 0.1], (len(points), 1))


def test_rotation_follows_its_circle():
    x0 = np.array([[1.0, 0.0, 0.5], [0.3, -0.8, -1.0]])
    for line in sl.lines(rotation, x0):
        t, x = line["time"], line["x"]
        s = x0[0] if np.isclose(x[np.argmin(np.abs(t)), 2], 0.5) else x0[1]
        exact = np.stack([s[0] * np.cos(t) - s[1] * np.sin(t), s[0] * np.sin(t) + s[1] * np.cos(t),
                          np.full_like(t, s[2])], axis=1)
        assert np.abs(x - exact).max() < 1e-6  # rel_err 1e-6 per step, a handful of steps
        assert line["status"] == (sl.REACHED, sl.REACHED)
        assert np.allclose(line["val"], rotation(x), rtol=0, atol=1e-15)


def test_linear_shear_is_integrated_exactly():
    # x(t) = x0 + rate y0 t: a polynomial of degree one, which every Runge-Kutta stage reproduces
    x0 = np.array([[0.2, 1.5, -0.4]])
    (line,) = sl.lines(shear, x0, t_final=2.0)
    t, x = line["time"], line["x"]
    exact = x0[0][None, :] + np.outer(t, [0.7 * 1.5, 0.0, 0.0])
    assert np.abs(x - exact).max() < 1e-13
    assert t[0] == -2.0 and t[-1] == 2.0


def test_constant_flow_step_sequence():
    # k_i = c for every stage: the error estimate is 0 (sum b = sum b* = 1), every try is accepted and dt grows by
    # 0.9 * (5^-5)^(-1/5) = 4.5 until it is cut to land on t_final: t = 0, 0.1, 0.55, 1.0
    trace = []
    x, t, v, st = sl.integrate(lambda p: constant(p[None])[0], lambda p: constant(p[None])[0], np.zeros(3), 1.0, 0.1,
                               1e-10, 1e-6, trace=trace)
    assert st == sl.REACHED
    assert np.allclose(t, [0.0, 0.1, 0.55, 1.0], rtol=0, atol=1e-15)
    assert [a for *_, a in trace] == [True, True, True]
    dts = [d for _, d, _, _ in trace]
    assert dts[0] == 0.1 and abs(dts[1] - 0.45) < 1e-15 and abs(dts[2] - (1.0 - t[2])) == 0.0
    assert np.allclose(x, np.outer(t, [0.3, -0.2, 0.1]), rtol=0, atol=1e-15)


def test_rejected_step_shrinks_dt_by_the_formula():
    # v = (1, 0, 0) below x = 0.05, (1, s, 0) beyond it.  From the origin with dt = 0.1 the stage points lie at
    # x = 0, 0.02, 0.03, 0.06, 0.1, 0.0875 (c_i dt): stages 4-6 see s.  Then y_err = dt s (db_4 + db_5 + db_6),
    # |x| = 0 and k1_y = 0, so err = |y_err| / abs_err; it is rejected and dt becomes dt * max(0.9 err^(-1/3), 0.2)
    s, abs_err = 2.0, 1e-3

    def step_flow(p):
        return np.array([1.0, s if p[0] > 0.05 else 0.0, 0.0])

    trace = []
    sl.integrate(step_flow, step_flow, np.zeros(3), 1.0, 0.1, abs_err, 0.0, trace=trace)
    db = [125 / 594 - 13525 / 55296, 0 - 277 / 14336, 512 / 1771 - 1 / 4]
    err = abs(0.1 * s * sum(db)) / abs_err
    assert err > 1.0
    t0, dt0, err0, ok0 = trace[0]
    assert (t0, dt0, ok0) == (0.0, 0.1, False)
    assert err0 == pytest.approx(err, rel=1e-12)
    assert trace[1][1] == pytest.approx(0.1 * max(0.9 * err ** (-1 / 3), 0.2), rel=1e-12)


def test_lands_exactly_on_t_final_both_ways():
    for T in (1.0, 0.37, 3.1):
        (line,) = sl.lines(rotation, [[0.4, 0.2, 0.0]], t_final=T, dt_init=0.07)
        assert abs(line["time"][-1] - T) <= sl.DBL_EPSILON
        assert abs(line["time"][0] + T) <= sl.DBL_EPSILON


def test_back_and_forward_join():
    x0 = np.array([0.4, 0.2, 0.0])
    vel1 = lambda p: rotation(p[None])[0]  # noqa: E731
    bx, bt, _, _ = sl.integrate(vel1, vel1, x0, -1.0, -0.1, 1e-10, 1e-6)
    fx, ft, _, _ = sl.integrate(vel1, vel1, x0, 1.0, 0.1, 1e-10, 1e-6)
    (line,) = sl.lines(rotation, [x0])
    t, x = line["time"], line["x"]
    assert len(t) == len(bt) + len(ft) - 1
    assert np.all(np.diff(t) > 0)
    assert np.array_equal(t[:len(bt) - 1], bt[:0:-1]) and np.array_equal(t[len(bt) - 1:], ft)
    assert np.array_equal(x[len(bt) - 1], x0) and np.count_nonzero(t == 0.0) == 1
    assert np.array_equal(x[:len(bt) - 1], bx[:0:-1])
    (fwd,) = sl.lines(rotation, [x0], back_integrate=False)
    assert np.array_equal(fwd["time"], ft) and fwd["status"] == (sl.REACHED, sl.REACHED)


def test_zero_tolerances_end_after_500_failures():
    # abs_err = rel_err = 0: every error with a nonzero estimate is infinite and every try fails, dt shrinking by 0.2.
    # On a smooth flow the estimate becomes exactly 0 once dt is below x's rounding (all six stages at x), and the
    # line creeps on instead; a flow that jumps at the seed x = 0 keeps it nonzero down to subnormal stage offsets,
    # which a dt of 1e100 does not reach within 500 tries
    def jump(p):
        return np.array([1.0 if p[0] <= 0.0 else 2.0, 0.5, 0.0])

    trace = []
    x, t, _, st = sl.integrate(jump, jump, np.zeros(3), 1e100, 1e100, 0.0, 0.0, trace=trace)
    assert st == sl.FAILED and len(trace) == sl.MAX_FAILS and len(x) == 1
    assert all(e == np.inf and not ok for _, _, e, ok in trace)
    assert trace[1][1] == 1e100 * 0.2 and trace[2][1] == 1e100 * 0.2 * 0.2
    (line,) = sl.lines(lambda p: np.array([jump(q) for q in p]), np.zeros((1, 3)), t_final=1e100, dt_init=1e100,
                       abs_err=0.0, rel_err=0.0, back_integrate=False)
    assert line["status"] == (sl.REACHED, sl.FAILED) and len(line["time"]) == 1


def test_max_points_caps_a_direction():
    (line,) = sl.lines(rotation, [[0.4, 0.2, 0.0]], max_points=3)
    assert line["status"] == (sl.CAPPED, sl.CAPPED) and len(line["time"]) == 5


def test_singular_seed_keeps_its_point():
    fast = lambda p: 2e3 * rotation(p)  # noqa: E731
    (line,) = sl.lines(fast, [[1.0, 0.0, 0.0]])
    assert line["status"] == (sl.SINGULAR, sl.SINGULAR) and len(line["time"]) == 1


def test_vorticity_of_a_linear_flow_is_its_curl():
    rng = np.random.default_rng(3)
    M = rng.normal(size=(3, 3))
    lin = lambda p: np.asarray(p) @ M.T  # noqa: E731  v = M r
    curl = np.array([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]])
    for x in rng.uniform(-1, 1, (5, 3)):
        w = sl.vorticity(lin, x)
        assert np.abs(w - curl).max() < 1e-7 * np.abs(curl).max()
    # a vortex line of a rigid rotation (uniform vorticity 2 e_z) is a straight vertical line
    (line,) = sl.lines(rotation, [[0.3, 0.1, 0.0]], kind=1)
    assert np.allclose(line["x"][:, :2], [0.3, 0.1], atol=1e-8)
    assert np.allclose(line["x"][:, 2], 2.0 * line["time"], atol=1e-7)

"""GPU tests of the listener (include/skelly_b200_flow.h: skb_flow_set_listener_frame, skb_flow_listener_velocity,
skb_flow_listener_lines): the velocity field against the oracle's flows with the body-interior replacement, and the
device's lockstep streamlines and vortex lines against tests/streamline_reference.py driven by the oracle's velocity."""
import numpy as np
import pytest

import oracle as orc
import skellysim_b200 as skb
import streamline_reference as sl
from conftest import rel_l2, rel_max
from test_gpu_flow import ft_of, load, make_system

pytestmark = pytest.mark.gpu
ETA = 0.9


def rigid_motion(r, center, uw):
    # U + omega x dx, one rounding per operation as the reference's Eigen expression
    dx = r - center
    w = uw[3:]
    return uw[:3] + np.stack([w[1] * dx[:, 2] - w[2] * dx[:, 1], w[2] * dx[:, 0] - w[0] * dx[:, 2],
                              w[0] * dx[:, 1] - w[1] * dx[:, 0]], axis=1)


class Frame:
    """A system as test_gpu_flow.make_system builds it, its frame and the oracle's velocity with the interior
    replacement (System::velocity_at_targets, system.cpp:330-384)."""

    def __init__(self, seed=5, n_fibers=6, n_shell=200, n_body_nodes=120, n_bodies=2, points=True, background=True):
        self.fib, self.shell, self.body = make_system(seed, n_fibers, n_shell, n_body_nodes, n_bodies)
        rng = np.random.default_rng(seed + 100)
        self.kind = np.array([1, 2] * n_bodies, dtype=np.int32)[:n_bodies]
        self.radii = np.tile([0.4, 0.5, 0.3], (n_bodies, 1))
        self.uw = rng.uniform(-0.5, 0.5, (n_bodies, 6))
        self.pts = rng.uniform(-1, 1, (2, 3)) if points else np.zeros((0, 3))
        self.pf, self.ptq = 0.3 * rng.normal(size=(len(self.pts), 3)), 0.3 * rng.normal(size=(len(self.pts), 3))
        self.bg = ([1, 0, 2], np.array([0.2, -0.1, 0.05]), np.array([0.05, 0.0, -0.02])) if background else None

    def open(self):
        fl = skb.Flow(0)
        load(fl, self.fib, self.shell, self.body)
        if len(self.pts):
            fl.set_point_sources(self.pts, self.pf, self.ptq)
        if self.bg:
            fl.set_background(*self.bg)
        fl.set_listener_frame(self.fib["forces"], self.shell["density"], self.body["density"], ft_of(self.body),
                              self.uw, self.kind, self.radii, ETA)
        return fl

    def flow(self, r):
        fib, shell, body = self.fib, self.shell, self.body
        v = orc.fiber_flow(r, fib["pos"], fib["n_nodes"], fib["lengths"], fib["forces"], ETA, subtract_self=False)
        v += orc.periphery_flow(r, shell["pos"], shell["normals"], shell["density"], ETA)
        if len(body["centers"]):
            v += orc.body_flow(r, body["pos"], body["normals"], body["density"], body["centers"], body["forces"],
                               body["torques"], ETA)
        if len(self.pts):
            v += orc.oseen_contract(self.pts, r, self.pf, ETA) + orc.rotlet(self.pts, r, self.ptq, ETA)
        if self.bg:
            comp, scale, uni = self.bg
            v += uni[None, :] + r[:, comp] * scale[None, :]
        return v

    def inside(self, r):
        """per body, the points its interior test takes (library order: the last match wins)"""
        out = []
        for b, c in enumerate(self.body["centers"]):
            dx = r - c
            if self.kind[b] == 1:
                out.append(np.sqrt(dx[:, 0] * dx[:, 0] + dx[:, 1] * dx[:, 1] + dx[:, 2] * dx[:, 2]) < self.radii[b, 0])
            else:
                q = [dx[:, j] * dx[:, j] / self.radii[b, j] / self.radii[b, j] for j in range(3)]
                out.append(q[0] + q[1] + q[2] < 1.0)
        return out

    def velocity(self, r):
        r = np.asarray(r, dtype=np.float64)
        v = self.flow(r)
        for b, m in enumerate(self.inside(r)):
            v[m] = rigid_motion(r[m], self.body["centers"][b], self.uw[b])
        return v


def seeds(rng, n, box=2.5):
    return rng.uniform(-box, box, (n, 3))


def clear_seeds(fr, rng, n, box=2.0, gap=0.4):
    """seeds at least `gap` from every source node and point source: lines that neither graze a singular Stokeslet
    nor creep along one, so that the device and the restatement take the same accept / reject decisions"""
    nodes = np.concatenate([fr.fib["pos"], fr.shell["pos"], fr.body["pos"], fr.pts, fr.body["centers"]])
    out = []
    while len(out) < n:
        x = rng.uniform(-box, box, 3)
        if len(nodes) == 0 or np.linalg.norm(nodes - x, axis=1).min() > gap:
            out.append(x)
    return np.array(out)


def test_velocity_field_matches_the_oracle_with_the_interior_replacement():
    fr = Frame()
    rng = np.random.default_rng(0)
    c = fr.body["centers"]
    r = np.concatenate([seeds(rng, 700), c[0] + rng.uniform(-0.2, 0.2, (40, 3)),
                        c[1] + rng.uniform(-0.25, 0.25, (40, 3)) * [1.0, 0.6, 0.7]])
    with fr.open() as fl:
        v = fl.velocity_field(r)
    ins = fr.inside(r)
    assert ins[0][700:740].all() and ins[1][740:].all()
    ref = fr.velocity(r)
    free = ~(ins[0] | ins[1])
    assert rel_max(v[free], ref[free]) < 1e-12 and rel_l2(v[free], ref[free]) < 1e-12
    assert np.array_equal(v[~free], ref[~free])  # exactly U + omega x dx


def test_background_only_streamlines_match_the_restatement():
    fr = Frame(n_fibers=0, n_shell=0, n_body_nodes=0, n_bodies=0, points=False)
    x0 = seeds(np.random.default_rng(1), 5, 1.0)
    with fr.open() as fl:
        got = fl.streamlines(x0)
    ref = sl.lines(fr.velocity, x0, max_points=1000)
    for g, e in zip(got, ref):
        assert len(g["time"]) == len(e["time"]) and g["status"] == e["status"]
        assert np.abs(g["x"] - e["x"]).max() <= 1e-12 * max(1.0, np.abs(e["x"]).max())
        assert np.abs(g["time"] - e["time"]).max() <= 1e-12


def _step_check(fr, line, kind, tol_x):
    # every returned step, re-run by the restatement from the device's x_i with the device's dt_i: lands on x_{i+1}
    # with err <= 1 (a start at the point nearer t = 0: the back points come reversed)
    vel1 = lambda x: fr.velocity(x[None])[0]  # noqa: E731
    deriv = vel1 if kind == 0 else (lambda x: sl.vorticity(fr.velocity, x))
    x, t = line["x"], line["time"]
    for i in range(len(t) - 1):
        a, b = (i, i + 1) if abs(t[i]) < abs(t[i + 1]) or t[i] == 0 else (i + 1, i)
        x_new, err, _ = sl.cash_karp_step(deriv, x[a], t[b] - t[a], 1e-10, 1e-6)
        assert err <= 1.0 + 1e-6, (i, err)
        assert np.abs(x_new - x[b]).max() <= tol_x * max(1.0, np.abs(x[b]).max()), i


@pytest.mark.parametrize("kind", [0, 1])
def test_full_flow_lines_match_the_restatement(kind):
    fr = Frame()
    x0 = clear_seeds(fr, np.random.default_rng(21), 4)
    with fr.open() as fl:
        got = fl.streamlines(x0) if kind == 0 else fl.vortexlines(x0)
    ref = sl.lines(fr.velocity, x0, kind=kind, max_points=1000)
    for g, e in zip(got, ref):
        assert len(g["time"]) == len(e["time"]) and g["status"] == e["status"]
        assert np.all(np.diff(g["time"]) > 0)
        scale = max(1.0, np.abs(e["x"]).max())
        if kind == 0:
            assert np.abs(g["x"] - e["x"]).max() <= 1e-9 * scale
            assert np.abs(g["time"] - e["time"]).max() <= 1e-9 * scale
            assert np.abs(g["val"] - e["val"]).max() <= 1e-9 * max(1.0, np.abs(e["val"]).max())
            _step_check(fr, g, kind, 1e-8)
            continue
        # vortex lines: the vorticity's differences over 2e-7 carry ~1e-9 of the velocities' rounding, enough to flip a
        # borderline accept and move the intermediate points (by up to the step's local error); the lines' ends at
        # +-t_final, every step (re-run from the device's own points) and the vorticity at every point still agree
        assert np.abs(g["x"][[0, -1]] - e["x"][[0, -1]]).max() <= 1e-6 * scale
        assert abs(g["time"][0] - e["time"][0]) <= 4e-16 and abs(g["time"][-1] - e["time"][-1]) <= 4e-16
        w = np.array([sl.vorticity(fr.velocity, p) for p in g["x"]])
        assert np.abs(g["val"] - w).max() <= 1e-5 * max(1.0, np.abs(w).max())
        _step_check(fr, g, kind, 1e-6)


def test_exit_statuses_match_the_restatement():
    fr = Frame()
    cases = [(dict(abs_err=0.0, rel_err=0.0, max_points=40), clear_seeds(fr, np.random.default_rng(3), 2)),
             (dict(max_points=3), clear_seeds(fr, np.random.default_rng(4), 3))]
    with fr.open() as fl:
        for req, x0 in cases:
            got = fl.streamlines(x0, **req)
            ref = sl.lines(fr.velocity, x0, **req)
            for g, e in zip(got, ref):
                assert g["status"] == e["status"] and len(g["time"]) == len(e["time"]), (req, g["status"], e["status"])
    assert got[0]["status"] == (sl.CAPPED, sl.CAPPED) and len(got[0]["time"]) == 5
    # a strong point force: |v| > 1e3 at a seed beside it (the point is kept), an ordinary seed unaffected
    fr.pf = fr.pf.copy()
    fr.pf[0] = [4e3, 0.0, 0.0]
    x0 = np.stack([fr.pts[0] + 2e-5, clear_seeds(fr, np.random.default_rng(5), 1)[0]])
    with fr.open() as fl:
        got = fl.streamlines(x0)
    ref = sl.lines(fr.velocity, x0, max_points=1000)
    assert got[0]["status"] == (sl.SINGULAR, sl.SINGULAR) and len(got[0]["time"]) == 1
    for g, e in zip(got, ref):
        assert g["status"] == e["status"] and len(g["time"]) == len(e["time"])


def test_a_line_in_a_batch_matches_it_alone():
    fr = Frame()
    x0 = clear_seeds(fr, np.random.default_rng(6), 1000)
    with fr.open() as fl:
        batch = fl.streamlines(x0)
        for i in (0, 417, 999):
            (alone,) = fl.streamlines(x0[i:i + 1])
            assert len(alone["time"]) == len(batch[i]["time"]) and alone["status"] == batch[i]["status"]
            assert np.abs(alone["x"] - batch[i]["x"]).max() <= 1e-9 * max(1.0, np.abs(alone["x"]).max())


def test_repeated_calls_are_bitwise_identical():
    fr = Frame()
    x0 = seeds(np.random.default_rng(7), 50, 2.0)
    with fr.open() as fl:
        for f in (fl.streamlines, fl.vortexlines):
            a, b = f(x0), f(x0)
            for p, q in zip(a, b):
                for k in ("x", "time", "val"):
                    assert np.array_equal(p[k], q[k])
                assert p["status"] == q["status"]


def test_velocity_at_targets_after_lines_uses_its_own_targets():
    fr = Frame()
    r = seeds(np.random.default_rng(8), 1, 1.0)
    args = (fr.fib["forces"], fr.shell["density"], fr.body["density"], ft_of(fr.body), ETA)
    with fr.open() as fl:
        v1 = [fl.velocity_at_targets(r, *args) for _ in range(3)]  # direct, captured, replayed
        fl.streamlines(seeds(np.random.default_rng(9), 3, 1.0))
        v2 = fl.velocity_at_targets(r, *args)
        fl.velocity_field(seeds(np.random.default_rng(10), 1, 1.0))
        v3 = fl.velocity_at_targets(r, *args)
    assert np.array_equal(v1[0], v1[2]) and np.array_equal(v1[0], v2) and np.array_equal(v1[0], v3)


def _err(fn, code):
    with pytest.raises(skb.SkbError, match=f"error {code}:"):
        fn()


def test_refusals():
    import ctypes as C
    from skellysim_b200 import capi
    fr = Frame()
    x0 = seeds(np.random.default_rng(11), 2, 1.0)
    L = capi.library()
    with skb.Flow(0) as fl:
        load(fl, fr.fib, fr.shell, fr.body)
        _err(lambda: fl.streamlines(x0), 4)      # no frame
        _err(lambda: fl.velocity_field(x0), 4)
    with fr.open() as fl:
        _err(lambda: fl.streamlines(x0, dt_init=0.0), 1)
        _err(lambda: fl.streamlines(x0, dt_init=-0.1), 1)
        _err(lambda: fl.streamlines(x0, t_final=-1.0), 1)
        _err(lambda: fl.streamlines(x0, abs_err=-1e-3), 1)
        _err(lambda: fl.streamlines(x0, rel_err=-1e-3), 1)
        _err(lambda: fl.streamlines(x0, max_points=0), 1)
        for field in ("dt_init", "t_final", "abs_err", "rel_err"):
            _err(lambda: fl.streamlines(x0, **{field: np.nan}), 1)
            _err(lambda: fl.streamlines(x0, **{field: np.inf}), 1)
        bad = x0.copy()
        bad[1, 2] = np.nan
        _err(lambda: fl.vortexlines(bad), 1)
        _err(lambda: fl._lines(2, x0, 0.1, 1.0, 1e-10, 1e-6, True, 10), 1)
        req = capi.LineRequest(0.1, 1.0, 1e-10, 1e-6, 1, 10)
        out = np.zeros(100)
        i32 = np.zeros(10, dtype=np.int32)
        p, pi = out.ctypes.data_as(capi._dp), i32.ctypes.data_as(C.POINTER(C.c_int32))
        x0p = x0.ctypes.data_as(capi._dp)
        for args in [(None, C.byref(req), p, p, p, pi, pi), (x0p, None, p, p, p, pi, pi), (x0p, C.byref(req), None, p, p, pi, pi),
                     (x0p, C.byref(req), p, p, p, None, pi), (x0p, C.byref(req), p, p, p, pi, None)]:
            a, r, x, t, v, n, s = args
            assert L.skb_flow_listener_lines(fl._h, 0, a, 2, r, x, t, v, n, s) == 1
        assert L.skb_flow_listener_lines(fl._h, 0, x0p, -1, C.byref(req), p, p, p, pi, pi) == 1
        assert L.skb_flow_listener_lines(fl._h, 0, None, 0, None, None, None, None, None, None) == 0
        assert fl.streamlines(np.zeros((0, 3))) == []
        # the frame goes stale with the geometry, the point sources and the background flow
        fl.set_background(*fr.bg)
        _err(lambda: fl.streamlines(x0), 4)
        _err(lambda: fl.velocity_field(x0), 4)
        fl.set_listener_frame(fr.fib["forces"], fr.shell["density"], fr.body["density"], ft_of(fr.body), fr.uw,
                              fr.kind, fr.radii, ETA)
        fl.streamlines(x0)
        fl.set_point_sources(fr.pts, fr.pf, fr.ptq)
        _err(lambda: fl.vortexlines(x0), 4)
        _err(lambda: fl.set_listener_frame(fr.fib["forces"], fr.shell["density"], fr.body["density"], ft_of(fr.body),
                                           fr.uw, [3, 1], fr.radii, ETA), 1)


@pytest.mark.parametrize("shape", [(0, 150, 0, 0), (5, 0, 0, 0), (0, 0, 80, 1), (0, 0, 0, 0)])
def test_flows_with_empty_classes(shape):
    fr = Frame(8, *shape, points=False)
    x0 = clear_seeds(fr, np.random.default_rng(12), 3)
    with fr.open() as fl:
        v = fl.velocity_field(x0)
        got = fl.streamlines(x0, max_points=50)
    ref_v = fr.velocity(x0)
    assert np.abs(v - ref_v).max() <= 1e-12 * max(1.0, np.abs(ref_v).max())
    ref = sl.lines(fr.velocity, x0, max_points=50)
    for g, e in zip(got, ref):
        assert g["status"] == e["status"] and len(g["time"]) == len(e["time"])

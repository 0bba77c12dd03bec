"""GPU tests of skb_flow_listener_gradient (capi.listener_gradient): the velocity gradient and the pressure of the
listener's frame against the long-double restatement of tests/gradient_reference.py, source class by class and
for a whole frame; the frame of a step against the same frame from its parts; the rigid gradient inside bodies; the
vorticity of the existing vortex-line request; reproducibility; the following velocity calls; staleness and refusals.

Bound, target row by target row.  Every output of a pair is a short chain of FP64 operations whose parts are bounded
by m = 6 c |f| / r^2 (Stokeslet, Oseen), 8 |kappa| |S| / r^3 (stresslet) and 4 c |L| / r^3 (rotlet), each with a
relative error below 32 u (u = 2^-53: the 1/r seed's Newton step and at most ten roundings).  One split of the plain
kernel sums its sources in order, the reduction adds the splits in order and scales once: the error of a target's row
is below (n_src + 64) u M, M = sum over sources of m.  The pressure's parts are bounded by 2 eta m."""
import numpy as np
import pytest

import gradient_reference as gr
import pair_sum_reference as ps
import skellysim_b200 as skb
from skellysim_b200 import capi
from test_gpu_flow import ft_of, load
from test_gpu_listener import ETA, Frame, clear_seeds, seeds
from test_gpu_listener_state import make, opened, set_state, targets

pytestmark = pytest.mark.gpu
U = 2.0 ** -53


def reference(fr, r):
    """(G, p) of the restatement, the interior rows replaced as gradient_finish_kernel replaces them"""
    (ext, _, _), inside, rigid = gr.listener_gradient(fr.fib, fr.shell, fr.body, r, ETA, fr.kind, fr.radii, fr.uw,
                                                      (fr.pts, fr.pf, fr.ptq), fr.bg)
    ext = np.asarray(ext, dtype=np.float64)
    ext[inside] = rigid[inside]
    return gr.as_grad_pressure(ext)


def _inv_r(src, r, p):
    src = np.asarray(src, dtype=np.float64).reshape(-1, 3)
    if len(src) == 0:
        return np.zeros((len(r), 0))
    d = np.sqrt(((r[:, None, :] - src[None, :, :]) ** 2).sum(-1))
    with np.errstate(divide="ignore"):
        return np.where(d == 0, 0.0, 1.0 / d ** p)  # (1 / D of a regularised kernel is below 1 / r)


def magnitude(fr, r):
    """(M per target, n_src): the bound's sum of part magnitudes over every source of the frame"""
    c = 1.0 / (8 * np.pi * ETA)
    fib, shell, body = fr.fib, fr.shell, fr.body
    M = np.zeros(len(r))
    n = 0
    if len(fib["n_nodes"]):
        w = ps.trapezoid_weights(fib["n_nodes"], fib["lengths"])
        M += 6 * c * _inv_r(fib["pos"], r, 2) @ (np.linalg.norm(fib["forces"], axis=1) * w)
        n += len(w)
    for pos, nrm, rho in ((shell["pos"], shell["normals"], shell.get("density")),
                          (body["pos"], body["normals"], body.get("density"))):
        if len(pos):
            S = np.linalg.norm(2 * ETA * np.asarray(nrm)[:, :, None] * np.asarray(rho)[:, None, :], axis=(1, 2))
            M += 8 * (3 * c) * _inv_r(pos, r, 3) @ S
            n += len(pos)
    if len(body["centers"]):
        M += 6 * c * _inv_r(body["centers"], r, 2) @ np.linalg.norm(body["forces"], axis=1)
        M += 4 * c * _inv_r(body["centers"], r, 3) @ np.linalg.norm(body["torques"], axis=1)
        n += 2 * len(body["centers"])
    if len(fr.pts):
        M += 6 * c * _inv_r(fr.pts, r, 2) @ np.linalg.norm(fr.pf, axis=1)
        M += 4 * c * _inv_r(fr.pts, r, 3) @ np.linalg.norm(fr.ptq, axis=1)
        n += 2 * len(fr.pts)
    if fr.bg is not None:
        M += np.abs(fr.bg[1]).max()
    return M, n


def check_rows(fr, r, G, p, free):
    Gr, pr = reference(fr, r)
    M, n = magnitude(fr, r)
    tol = (n + 64) * U * M + 1e-300
    errG = np.abs(G - np.asarray(Gr, dtype=np.float64)).reshape(len(r), 9).max(axis=1)
    errp = np.abs(p - np.asarray(pr, dtype=np.float64))
    bad = np.flatnonzero(free & ((errG > tol) | (errp > 2 * ETA * tol)))
    assert bad.size == 0, (bad[:5], errG[bad[:5]], errp[bad[:5]], tol[bad[:5]])


CLASSES = {
    # (n_fibers, n_shell, n_body_nodes, n_bodies, points, background): counts that give the plain kernel a partial
    # last tile of sources and, against 333 targets, several source splits
    "fibers": (70, 0, 0, 0, False, False),
    "periphery": (0, 2900, 0, 0, False, False),
    "bodies": (0, 0, 1300, 2, False, False),
    "points": (0, 0, 0, 0, True, False),
    "background": (0, 0, 0, 0, False, True),
    "frame": (40, 1500, 600, 2, True, True),
}


@pytest.mark.parametrize("n_trg", [1, 333, 4099])
@pytest.mark.parametrize("cls", list(CLASSES))
def test_each_source_class_and_a_frame_match_the_restatement(cls, n_trg):
    nf, ns, nb_nodes, nb, pts, bg = CLASSES[cls]
    fr = Frame(21, nf, ns, nb_nodes, nb, points=pts, background=bg)
    fr.kind[:] = 0  # no interior test: every target is a fluid point
    r = seeds(np.random.default_rng(n_trg), n_trg, 3.0)
    with fr.open() as fl:
        G, p = capi.listener_gradient(fl, r)
    assert G.shape == (n_trg, 3, 3) and p.shape == (n_trg,)
    check_rows(fr, r, G, p, np.ones(n_trg, dtype=bool))


def test_inside_bodies_the_gradient_is_rigid_and_the_pressure_nan():
    fr = Frame()
    rng = np.random.default_rng(3)
    c = fr.body["centers"]
    r = np.concatenate([seeds(rng, 400, 2.5), c[0] + rng.uniform(-0.2, 0.2, (50, 3)),
                        c[1] + rng.uniform(-0.2, 0.2, (50, 3))])
    with fr.open() as fl:
        G, p = capi.listener_gradient(fl, r)
    ins = fr.inside(r)
    free = ~np.any(ins, axis=0)
    check_rows(fr, r, G, p, free)
    for b, m in enumerate(ins):
        last = m.copy()
        for later in ins[b + 1:]:
            last &= ~later
        assert last.any()
        w = fr.uw[b, 3:]
        rigid = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
        assert np.array_equal(G[last], np.broadcast_to(rigid, G[last].shape))
        assert np.isnan(p[last]).all()
    assert np.isfinite(p[free]).all()


def test_the_vorticity_matches_the_vortex_lines_differences():
    """No oracle: the antisymmetric part of the analytic gradient against the central differences (+-1e-7) that the
    vortex-line request reports at its seed"""
    fr = Frame(7, points=True, background=True)
    fr.kind[:] = 0
    x0 = clear_seeds(fr, np.random.default_rng(4), 20)
    with fr.open() as fl:
        G, _ = capi.listener_gradient(fl, x0)
        lines = fl.vortexlines(x0, back_integrate=False, max_points=1)
    w = np.stack([G[:, 2, 1] - G[:, 1, 2], G[:, 0, 2] - G[:, 2, 0], G[:, 1, 0] - G[:, 0, 1]], axis=1)
    fd = np.array([ln["val"][0] for ln in lines])
    scale = np.abs(G).reshape(len(x0), 9).max(axis=1)
    assert (np.abs(w - fd).max(axis=1) <= 1e-6 * scale).all(), np.abs(w - fd).max(axis=1) / scale


def test_two_calls_are_bitwise_equal_and_the_velocity_calls_unchanged():
    fr = Frame()
    rng = np.random.default_rng(5)
    r_g, r_v = seeds(rng, 700, 2.5), seeds(rng, 90, 2.5)
    args = (fr.fib["forces"], fr.shell["density"], fr.body["density"], ft_of(fr.body), ETA)
    with fr.open() as fl:
        v0, w0 = fl.velocity_field(r_v), fl.velocity_at_targets(r_v, *args)
        w0b = fl.velocity_at_targets(r_v, *args)
    with fr.open() as fl:
        a = capi.listener_gradient(fl, r_g)
        b = capi.listener_gradient(fl, r_g)
        v1 = fl.velocity_field(r_v)
        w1 = fl.velocity_at_targets(r_v, *args)
        capi.listener_gradient(fl, r_v)
        w1b = fl.velocity_at_targets(r_v, *args)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1], equal_nan=True)
    assert np.array_equal(v0, v1) and np.array_equal(w0, w1) and np.array_equal(w0b, w1b)


def test_the_frame_of_a_step_is_the_frame_of_its_parts():
    sd = make(3, 9, 180, 120, 2, bound=False)
    off = np.concatenate([[0], np.cumsum(sd["fib"]["n_nodes"])])
    r = targets(sd, np.random.default_rng(1))
    with opened(sd) as fl:
        set_state(fl, sd, False)
        g_state = capi.listener_gradient(fl, r)
        packed = np.concatenate([np.concatenate([sd["fib"]["pos"][a:b].T.reshape(-1), sd["tension"][a:b]])
                                 for a, b in zip(off[:-1], off[1:])])
        fl.build_fiber_operators(*sd["params"], 1e-3, ETA)
        ff = fl.apply_fiber_force(packed)
        nf, ns = 4 * int(off[-1]), len(sd["shell"]["pos"])
        xs, xb = sd["x"][nf:nf + 3 * ns], sd["x"][nf + 3 * ns:]
        per = sd["body"]["n_nodes"][0]
        blocks = xb.reshape(2, 3 * per + 6)
        fl.set_listener_frame(ff, xs.reshape(-1, 3), blocks[:, :3 * per].reshape(-1, 3), np.zeros((2, 6)),
                              blocks[:, 3 * per:], sd["kind"], sd["radii"], ETA)
        g_frame = capi.listener_gradient(fl, r)
    assert np.array_equal(g_state[0], g_frame[0]) and np.array_equal(g_state[1], g_frame[1], equal_nan=True)


def _err(fn, code):
    with pytest.raises(skb.SkbError, match=f"error {code}:"):
        fn()


def test_staleness_refusals_and_no_targets():
    import ctypes as C
    fr = Frame()
    r = seeds(np.random.default_rng(6), 5, 1.0)
    L = capi.library()
    with skb.Flow(0) as fl:
        load(fl, fr.fib, fr.shell, fr.body)
        _err(lambda: capi.listener_gradient(fl, r), 4)  # no frame
    with fr.open() as fl:
        G, p = capi.listener_gradient(fl, np.zeros((0, 3)))
        assert G.shape == (0, 3, 3) and p.shape == (0,)
        out = np.zeros(9 * 5)
        rp, op = r.ctypes.data_as(capi._dp), out.ctypes.data_as(capi._dp)
        assert L.skb_flow_listener_gradient(fl._h, None, 5, op, op) == 1
        assert L.skb_flow_listener_gradient(fl._h, rp, 5, None, op) == 1
        assert L.skb_flow_listener_gradient(fl._h, rp, 5, op, None) == 1
        assert L.skb_flow_listener_gradient(fl._h, rp, -1, op, op) == 1
        assert L.skb_flow_listener_gradient(fl._h, None, 0, None, None) == 0
        assert L.skb_flow_listener_gradient(None, rp, 5, op, op) == 1
        # non-finite targets are computed, as by the velocity field
        bad = r.copy()
        bad[2, 0] = np.nan
        G, p = capi.listener_gradient(fl, bad)
        assert np.isnan(G[2]).any() and np.isfinite(G[[0, 1, 3, 4]]).all()
        fl.set_background(*fr.bg)
        _err(lambda: capi.listener_gradient(fl, r), 4)
        fl.set_listener_frame(fr.fib["forces"], fr.shell["density"], fr.body["density"], ft_of(fr.body), fr.uw,
                              fr.kind, fr.radii, ETA)
        capi.listener_gradient(fl, r)
        fl.set_point_sources(fr.pts, fr.pf, fr.ptq)
        _err(lambda: capi.listener_gradient(fl, r), 4)
        fl.set_listener_frame(fr.fib["forces"], fr.shell["density"], fr.body["density"], ft_of(fr.body), fr.uw,
                              fr.kind, fr.radii, ETA)
        fl.set_fibers(fr.fib["pos"], fr.fib["n_nodes"], fr.fib["lengths"])
        _err(lambda: capi.listener_gradient(fl, r), 4)


@pytest.mark.parametrize("shape", [(0, 150, 0, 0), (5, 0, 0, 0), (0, 0, 80, 1), (0, 0, 0, 0)])
def test_frames_with_empty_classes(shape):
    fr = Frame(8, *shape, points=False)
    fr.kind[:] = 0
    r = seeds(np.random.default_rng(12), 200, 2.5)
    with fr.open() as fl:
        G, p = capi.listener_gradient(fl, r)
    check_rows(fr, r, G, p, np.ones(len(r), dtype=bool))

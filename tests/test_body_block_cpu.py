"""CPU tests of tests/system_reference.py, the restatement of the body block and the fiber-body links of
System::apply_matvec that the GPU tests compare against, checked against the reference's own second statements:
SphericalBody::update_preconditioner assembles the same body operator that ::matvec applies (body_spherical.cpp:39-63,
104-126), and calculate_link_conditions' terms have closed forms for straight and cubic fibers."""
import numpy as np
import pytest

import system_reference as sr
from oracle.fiber_fd import compute_matrices


def sphere(n, radius, center, seed=0):
    rng = np.random.default_rng(seed)
    e = rng.normal(size=(n, 3))
    e /= np.linalg.norm(e, axis=1)[:, None]
    return center + radius * e, e, np.full(n, 4.0 * np.pi * radius**2 / n)


def bodies_of(n_nodes, radius=0.4, seed=0):
    rng = np.random.default_rng(seed)
    pos, nrm, w, cen = [], [], [], []
    for b, n in enumerate(n_nodes):
        c = rng.uniform(-2, 2, 3)
        p, e, wb = sphere(n, radius, c, seed + b + 1)
        pos.append(p), nrm.append(e), w.append(wb), cen.append(c)
    pos, nrm, w = np.concatenate(pos), np.concatenate(nrm), np.concatenate(w)
    ex, ey, ez = (np.concatenate(v) for v in zip(*[sr.singularity_vectors(p, e, wb) for p, e, wb in
                                                      zip(np.split(pos, np.cumsum(n_nodes)[:-1]),
                                                          np.split(nrm, np.cumsum(n_nodes)[:-1]),
                                                          np.split(w, np.cumsum(n_nodes)[:-1]))]))
    return dict(pos=pos, normals=nrm, centers=np.array(cen), n_nodes=list(n_nodes), weights=w, ex=ex, ey=ey, ez=ez)


NO_FIBERS = dict(pos=np.zeros((0, 3)), n_nodes=[], lengths=[])
NO_OPS = dict(n_nodes=[], A=[], force=[], D_1_0={}, P={}, xs=np.zeros((0, 3)), length_prev=[], plus=[], D_2_0={},
              D_3_0={})
NO_SHELL = dict(pos=np.zeros((0, 3)), normals=np.zeros((0, 3)))


@pytest.mark.parametrize("n_nodes", [(40,), (73,)])
def test_isolated_body_rows_equal_the_assembled_body_operator(n_nodes):
    """One body alone: its rows of A x are A_ x_body (A_ holds the body's self-interaction only, so a second body's
    flow would add to them)."""
    bodies = bodies_of(n_nodes)
    x = np.random.default_rng(3).normal(size=int(sum(3 * n + 6 for n in n_nodes)))
    res, _, _ = sr.system_apply_matvec(NO_FIBERS, NO_SHELL, bodies, NO_OPS, dict(body=[], site=[], rigidity=[]), None,
                                       x, 1.3)
    ref = []
    node_off, sol_off = np.concatenate([[0], np.cumsum(n_nodes)]), np.concatenate([[0], np.cumsum(3 * np.array(n_nodes) + 6)])
    for b, n in enumerate(n_nodes):
        sl = slice(node_off[b], node_off[b] + n)
        A = sr.body_operator(bodies["pos"][sl], bodies["normals"][sl], bodies["centers"][b], bodies["weights"][sl],
                             bodies["ex"][sl], bodies["ey"][sl], bodies["ez"][sl])
        ref.append(A @ x[sol_off[b]:sol_off[b + 1]])
    ref = np.concatenate(ref)
    assert np.abs(res - ref).max() <= 1e-13 * np.abs(ref).max()


def test_stresslet_times_normal_contracts_to_the_density_form():
    p, e, w = sphere(30, 0.5, np.zeros(3), 5)
    d = np.random.default_rng(6).normal(size=(30, 3))
    lhs = sr.stresslet_times_normal(p, e) @ d.reshape(-1)
    rhs = sr.stresslet_times_normal_times_density(p, e, d).reshape(-1)
    assert np.abs(lhs - rhs).max() <= 1e-13 * np.abs(rhs).max()


def fiber_system(n_nodes, bound, seed=0):
    """Fibers with the reference's derivative matrices, bound per `bound` (body index or -1) to bodies_of((30, 30))."""
    rng = np.random.default_rng(seed)
    bodies = bodies_of((30, 30), seed=seed)
    pos, xs, lengths = [], [], []
    for n in n_nodes:
        L = rng.uniform(0.5, 2.0)
        t = rng.normal(size=3)
        t /= np.linalg.norm(t)
        pos.append(rng.uniform(-1, 1, 3) + np.linspace(0, L, n)[:, None] * t + 0.05 * rng.normal(size=(n, 3)))
        xs.append(np.tile(t, (n, 1)))
        lengths.append(L)
    fib = dict(pos=np.concatenate(pos), n_nodes=list(n_nodes), lengths=lengths)
    ops = dict(xs=np.concatenate(xs), length_prev=list(rng.uniform(0.5, 2.0, len(n_nodes))),
               D_2_0={n: compute_matrices(n)["D_2_0"] for n in set(n_nodes)},
               D_3_0={n: compute_matrices(n)["D_3_0"] for n in set(n_nodes)})
    links = dict(body=np.array(bound), site=rng.uniform(-2, 2, (len(n_nodes), 3)),
                 rigidity=rng.uniform(0.5, 2.0, len(n_nodes)))
    x_f = rng.normal(size=4 * int(np.sum(n_nodes)))
    x_b = rng.normal(size=sum(3 * n + 6 for n in bodies["n_nodes"]))
    return fib, ops, links, bodies, x_f, x_b


def test_literal_and_intended_links_agree_when_bound_fibers_lead():
    fib, ops, links, bodies, x_f, x_b = fiber_system((16, 24, 32, 16, 24), [0, 1, 0, -1, -1])
    v_i, ft_i = sr.link_conditions(fib, ops, links, bodies, x_f, x_b)
    v_l, ft_l = sr.link_conditions(fib, ops, links, bodies, x_f, x_b, literal=True)
    assert np.array_equal(v_i, v_l) and np.array_equal(ft_i, ft_l)
    assert np.count_nonzero(v_i[3:]) == 0  # free fibers: zeros (body_container.cpp:177)


def test_literal_and_intended_links_differ_after_a_free_fiber():
    fib, ops, links, bodies, x_f, x_b = fiber_system((16, 16, 16), [-1, 0, 1])
    v_i, _ = sr.link_conditions(fib, ops, links, bodies, x_f, x_b)
    v_l, _ = sr.link_conditions(fib, ops, links, bodies, x_f, x_b, literal=True)
    assert np.count_nonzero(v_i[0]) == 0 and np.count_nonzero(v_l[2]) == 0  # the literal reading writes rows 0 and 1
    assert not np.allclose(v_i, v_l)


def test_straight_fiber_force_and_torque_are_the_tension_terms():
    fib, ops, links, bodies, x_f, x_b = fiber_system((16, 32), [0, 1], seed=2)
    # straight fibers in x_fibers: xss = xsss = 0
    off = 0
    for f, n in enumerate(fib["n_nodes"]):
        line = np.linspace(0, 1.3, n)[:, None] * np.array([0.6, 0.0, 0.8]) + np.array([0.1, -0.2, 0.3])
        x_f[4 * off:4 * off + 3 * n] = line.T.reshape(-1)
        off += n
    _, ft = sr.link_conditions(fib, ops, links, bodies, x_f, x_b)
    off = 0
    for f, n in enumerate(fib["n_nodes"]):
        xs0, T0 = ops["xs"][off], x_f[4 * off + 3 * n]
        b = links["body"][f]
        s = links["site"][f] - bodies["centers"][b]
        # rounding of (2/L)^3 sum_j x_j D_3_0(j, 0): the derivative of a straight line is zero only to that scale
        tol = 64 * np.finfo(float).eps * links["rigidity"][f] * (2.0 / fib["lengths"][f]) ** 3 * \
            np.abs(ops["D_3_0"][n][:, 0]).sum() * 2.0 * (1 + np.linalg.norm(s))
        assert np.abs(ft[b, :3] - xs0 * T0).max() <= tol
        assert np.abs(ft[b, 3:] - np.cross(s, xs0) * T0).max() <= tol
        off += n


def test_tension_condition_is_the_tangent_velocity():
    fib, ops, links, bodies, x_f, x_b = fiber_system((16, 24, 32), [0, 1, 0], seed=4)
    for seed in range(5):
        x_b = np.random.default_rng(seed).normal(size=x_b.shape)
        v, _ = sr.link_conditions(fib, ops, links, bodies, x_f, x_b)
        xs0 = ops["xs"][np.concatenate([[0], np.cumsum(fib["n_nodes"])[:-1]])]
        assert np.allclose(v[:, 3], np.einsum("fk,fk->f", xs0, v[:, :3]), rtol=0, atol=1e-13 * np.abs(v).max())
        vd, _ = sr.link_conditions(fib, ops, links, bodies, x_f, x_b, defect="omega_site_sign")
        assert not np.allclose(vd[:, 3], np.einsum("fk,fk->f", xs0, vd[:, :3]))  # the planted defect is caught


@pytest.mark.parametrize("defect", [None, "xsss_length_prev"])
def test_cubic_fiber_bending_terms(defect):
    """x(s) = x0 + (s, a s^2 / 2, b s^3 / 6): xss(0) = (0, a, 0), xsss(0) = (0, 0, b) exactly for the reference's
    (4 + k)-point stencils, so F = -E (0, 0, b) + xs0 T0 and L = -E s x (0, 0, b) + (s x xs0) T0 + E xs0 x (0, a, 0)."""
    fib, ops, links, bodies, x_f, x_b = fiber_system((24,), [1], seed=6)
    n, L, a, bb = 24, fib["lengths"][0], 0.7, -1.1
    s_nodes = (compute_matrices(n)["alpha"] + 1.0) * L / 2.0
    x0 = np.array([0.2, 0.1, -0.3])
    curve = x0 + np.stack([s_nodes, a * s_nodes**2 / 2, bb * s_nodes**3 / 6], axis=1)
    x_f[:3 * n] = curve.T.reshape(-1)
    ops["xs"][:] = (1.0, 0.0, 0.0)
    _, ft = sr.link_conditions(fib, ops, links, bodies, x_f, x_b, defect=defect)
    E, T0, xs0 = links["rigidity"][0], x_f[3 * n], np.array([1.0, 0.0, 0.0])
    s = links["site"][0] - bodies["centers"][1]
    xsss, xss = np.array([0.0, 0.0, bb]), np.array([0.0, a, 0.0])
    F = -E * xsss + xs0 * T0
    Lb = -E * np.cross(s, xsss) + np.cross(s, xs0) * T0 + E * np.cross(xs0, xss)
    ok = np.allclose(ft[1, :3], F, rtol=1e-9, atol=1e-9) and np.allclose(ft[1, 3:], Lb, rtol=1e-9, atol=1e-9)
    assert ok == (defect is None)  # length_ vs length_prev_ in xsss is caught

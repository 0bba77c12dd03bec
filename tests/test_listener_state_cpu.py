"""CPU tests of tests/listener_state_reference.py, the restatement the GPU tests of skb_flow_set_listener_state hold the
device to: pinned to the reference's own statements (a straight bound fiber loads its body with xs_0 T_0, free fibers
with nothing, no repulsion without the flag, no external force or torque), and every planted defect misses the 1e-12
gate by orders of magnitude."""
import numpy as np
import pytest

import listener_state_reference as lsr

N = 16
SHAPE = dict(kind="sphere", a=2.0, b=0.0, c=0.0, f_0=20.0, l_0=0.5, binding_active=0, polar_angle_start=0.0,
             polar_angle_end=np.pi, binding_threshold=0.75)


def system(seed=3, bound=(0, 1, -1), n_shell=12, body_nodes=(10, 14)):
    """three fibers near the periphery's surface (|x| ~ 1.7), two bodies, a random solution and tension"""
    rng = np.random.default_rng(seed)
    pos, lengths = [], []
    for f in range(len(bound)):
        t = rng.normal(size=3)
        t /= np.linalg.norm(t)
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        L = rng.uniform(0.3, 0.5)
        pos.append(1.5 * d + np.linspace(0.0, L, N)[:, None] * t)
        lengths.append(L)
    fib = dict(pos=np.concatenate(pos), n_nodes=[N] * len(bound), lengths=np.array(lengths))
    bodies = dict(n_nodes=list(body_nodes), centers=rng.uniform(-0.5, 0.5, (len(body_nodes), 3)))
    links = dict(body=np.array(bound), site=np.array([p[0] for p in pos]), rigidity=np.full(len(bound), 2.5e-3))
    n_x = 4 * N * len(bound) + 3 * n_shell + sum(3 * n + 6 for n in body_nodes)
    x = rng.uniform(-1, 1, n_x)
    tension = rng.uniform(-1, 1, N * len(bound))
    params = (fib["lengths"], 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)
    return fib, n_shell, bodies, links, params, x, tension


def run(sys_, **kw):
    fib, n_shell, bodies, links, params, x, tension = sys_
    kw.setdefault("shape", SHAPE)
    return lsr.frame(fib, n_shell, bodies, links, params, 1e-3, 0.9, x, tension, **kw)


def test_a_straight_bound_fiber_loads_its_body_with_xs0_T0():
    s = system(bound=(0,), body_nodes=(10,))
    fib, _, bodies, links, params, x, tension = s
    out = run(s)
    ops = lsr._operators(fib, params, 1e-3, 0.9)
    xs0, T0 = ops[0].xs[0], tension[0]
    site = links["site"][0] - bodies["centers"][0]
    F, L = out["body_ft"][0, :3], out["body_ft"][0, 3:]
    # xss and xsss of a straight fiber vanish up to the rounding of the finite differences
    assert np.abs(F - xs0 * T0).max() <= 1e-9 * abs(T0)
    assert np.abs(L - np.cross(site, xs0) * T0).max() <= 1e-9 * abs(T0)
    assert abs(np.linalg.norm(xs0) - 1.0) <= 1e-12


def test_free_fibers_give_exactly_zero_body_force():
    s = system(bound=(-1, -1, -1))
    assert np.array_equal(run(s)["body_ft"], np.zeros((2, 6)))
    fib, n_shell, bodies, _, params, x, tension = s
    assert np.array_equal(run((fib, n_shell, bodies, None, params, x, tension))["body_ft"], np.zeros((2, 6)))


def test_the_repulsion_enters_with_the_flag_only():
    s = system()
    fib, _, _, _, params, x, tension = s
    off, on = run(s), run(s, periphery_interaction=True)
    ops = lsr._operators(fib, params, 1e-3, 0.9)
    want = np.concatenate([(op.force_operator @ np.concatenate([fib["pos"][N * f:N * (f + 1)].T.reshape(-1),
                                                                tension[N * f:N * (f + 1)]])).reshape(3, N).T
                           for f, op in enumerate(ops)])
    assert np.array_equal(off["fib_forces"], want)
    assert np.abs(on["fib_forces"] - off["fib_forces"]).max() > 1e-3


def test_external_forces_and_torques_do_not_enter():
    s = system()
    ext = np.random.default_rng(1).uniform(-5, 5, (2, 6))
    a, b = run(s), run(s, external_ft=ext)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_the_densities_and_rigid_motions_are_the_solution_slices():
    s = system()
    fib, n_shell, bodies, _, _, x, _ = s
    out = run(s)
    nf = 4 * N * 3
    assert np.array_equal(out["shell_density"].reshape(-1), x[nf:nf + 3 * n_shell])
    xb = x[nf + 3 * n_shell:]
    assert np.array_equal(out["body_densities"][:10].reshape(-1), xb[:30])
    assert np.array_equal(out["body_uw"][0], xb[30:36])
    assert np.array_equal(out["body_densities"][10:].reshape(-1), xb[36:36 + 42])
    assert np.array_equal(out["body_uw"][1], xb[78:84])


@pytest.mark.parametrize("defect", lsr.DEFECTS)
def test_every_planted_defect_misses_the_gate_by_orders_of_magnitude(defect):
    s = system()
    ext = np.random.default_rng(2).uniform(-1, 1, (2, 6))
    fs = np.array([0.7, -0.4, 1.1])
    clean = run(s, external_ft=ext, force_scale=fs)
    bad = run(s, external_ft=ext, force_scale=fs, defect=defect)
    assert lsr.gate(clean, clean) == 0.0
    assert lsr.gate(bad, clean) > 1e-6, (defect, lsr.gate(bad, clean))

"""CPU tests of the physics of tests/gradient_reference.py, the restatement the GPU tests of skb_flow_listener_gradient
hold the device to: its gradients against long-double central differences of the oracle's velocities, class by class;
the pressure against the Stokes equations (grad p = eta lap u); the trace of the gradient; the interior rule and the
r == 0 rule; and the marshalling of capi.listener_gradient."""
import numpy as np
import pytest

import gradient_reference as gr
import oracle as orc
from skellysim_b200 import capi
from test_capi_binding_cpu import _drive, _inputs, _twin_calls, calls  # noqa: F401 (the fixture)

ETA = 0.7
LD = np.longdouble


def _system(seed, n_src=6):
    rng = np.random.default_rng(seed)
    src = rng.uniform(-1, 1, (n_src, 3))
    trg = rng.uniform(2, 3, (5, 3)) * rng.choice([-1, 1], (5, 3))  # well away from every source
    return rng, src, trg


def _fd_gradient(vel, r, h=1e-4):
    """central differences, d u_i / d x_j, of vel: (n, 3) -> (n, 3)"""
    G = np.zeros((len(r), 3, 3))
    for j in range(3):
        e = np.zeros(3)
        e[j] = h
        G[:, :, j] = (np.asarray(vel(r + e), dtype=LD) - np.asarray(vel(r - e), dtype=LD)) / (2 * LD(h))
    return G


def _G(part):
    return np.asarray(part[0][:, :9], dtype=LD).reshape(-1, 3, 3)


def _Gp(part, eta=ETA):
    """(G, p) of a part, its pressure multiplied by eta as gradient_finish_kernel does"""
    return _G(part), part[0][:, 9] * LD(eta)


def _sym6(S9):
    S9 = np.asarray(S9, dtype=np.float64).reshape(-1, 9)
    return np.stack([S9[:, 0], S9[:, 4], S9[:, 8], S9[:, 1] + S9[:, 3], S9[:, 2] + S9[:, 6], S9[:, 5] + S9[:, 7]], 1)


def stokeslet(src, f, r):
    return _Gp(gr.pair_grad_rows("sl", src, f, r, ETA))


def stresslet(src, S9, r):
    return _Gp(gr.pair_grad_rows("dl6", src, _sym6(S9), r, ETA))


def _flows(rng, src):
    f = rng.normal(size=src.shape)
    S = rng.normal(size=(len(src), 9))
    L = rng.normal(size=src.shape)
    return {
        "stokeslet": (lambda r: orc.stokeslet_direct_ld(src, f, r) / ETA, lambda r: stokeslet(src, f, r)[0]),
        "stresslet": (lambda r: orc.stresslet_direct_ld(src, S, r) / ETA, lambda r: stresslet(src, S, r)[0]),
        "rotlet": (lambda r: orc.rotlet(src, r, L, ETA), lambda r: _G(gr.rotlet_grad(r, src, L, ETA))),
        "oseen": (lambda r: orc.oseen_contract(src, r, f, ETA), lambda r: _G(gr.oseen_grad(r, src, f, ETA))),
    }


@pytest.mark.parametrize("kind", ["stokeslet", "stresslet", "rotlet", "oseen"])
def test_the_gradient_is_the_derivative_of_the_oracle_velocity(kind):
    rng, src, trg = _system(1)
    vel, grad = _flows(rng, src)[kind]
    G = np.asarray(grad(trg), dtype=np.float64)
    fd = _fd_gradient(vel, trg)
    assert np.abs(G - fd).max() <= 1e-7 * np.abs(G).max(), np.abs(G - fd).max() / np.abs(G).max()


def test_the_background_gradient_is_its_scale():
    comp, scale = [1, 0, 2], np.array([0.2, -0.1, 0.05])
    G = _G(gr.background_grad(2, comp, scale))
    expect = np.zeros((3, 3))
    expect[0, 1], expect[1, 0], expect[2, 2] = scale
    assert np.array_equal(G[0], expect) and np.array_equal(G[1], expect)


@pytest.mark.parametrize("kind", ["stokeslet", "stresslet"])
def test_the_pressure_satisfies_the_stokes_equations(kind):
    rng, src, trg = _system(2)
    f, S = rng.normal(size=src.shape), rng.normal(size=(len(src), 9))
    if kind == "stokeslet":
        gp = lambda r: stokeslet(src, f, np.asarray(r, dtype=np.float64))
    else:
        gp = lambda r: stresslet(src, S, np.asarray(r, dtype=np.float64))
    # lap u_i = d_j (d_j u_i): the Laplacian of the velocity from the analytic gradient's own divergence
    def lap_u(r):
        h = LD(1e-4)
        out = np.zeros((len(r), 3), dtype=LD)
        for j in range(3):
            e = np.zeros(3, dtype=LD)
            e[j] = h
            out += (gp(np.asarray(r, dtype=LD) + e)[0][:, :, j] - gp(np.asarray(r, dtype=LD) - e)[0][:, :, j]) / (2 * h)
        return out
    h = LD(1e-4)
    grad_p = np.stack([(gp(np.asarray(trg, dtype=LD) + e)[1] - gp(np.asarray(trg, dtype=LD) - e)[1]) / (2 * h)
                       for e in np.eye(3, dtype=LD) * h], axis=1)
    lhs = ETA * lap_u(trg)
    assert np.abs(grad_p - lhs).max() <= 1e-6 * np.abs(grad_p).max()


def test_the_trace_vanishes_where_the_flow_is_incompressible():
    rng, src, trg = _system(3)
    f, L = rng.normal(size=src.shape), rng.normal(size=src.shape)
    S = rng.normal(size=(len(src), 3, 3))
    S -= np.trace(S, axis1=1, axis2=2)[:, None, None] * np.eye(3) / 3
    for G in (stokeslet(src, f, trg)[0], _G(gr.rotlet_grad(trg, src, L, ETA)),
              stresslet(src, S.reshape(-1, 9), trg)[0]):
        tr = np.trace(np.asarray(G, dtype=np.float64), axis1=1, axis2=2)
        assert np.abs(tr).max() <= 1e-15 * np.abs(np.asarray(G, dtype=np.float64)).max()


def test_a_coincident_pair_adds_nothing():
    rng, src, trg = _system(4)
    f, S, L = rng.normal(size=src.shape), rng.normal(size=(len(src), 9)), rng.normal(size=src.shape)
    r = np.concatenate([trg, src[:2]])
    for fn in (lambda k, r: stokeslet(src[k], f[k], r), lambda k, r: stresslet(src[k], S[k], r),
               lambda k, r: _Gp(gr.oseen_grad(r, src[k], f[k], ETA)),
               lambda k, r: (_G(gr.rotlet_grad(r, src[k], L[k], ETA)), None)):
        all_src = fn(slice(None), r)
        # target src[0] against the other sources only equals the full sum there
        others = fn(slice(1, None), r[-2:-1])
        assert np.array_equal(all_src[0][-2], others[0][0])
        if all_src[1] is not None:
            assert all_src[1][-2] == others[1][0]


def test_the_interior_rule():
    body = dict(centers=np.array([[0.0, 0, 0], [0.1, 0, 0]]), pos=np.zeros((0, 3)), normals=np.zeros((0, 3)),
                density=np.zeros((0, 3)), forces=np.zeros((2, 3)), torques=np.zeros((2, 3)))
    empty = dict(pos=np.zeros((0, 3)), n_nodes=[], lengths=[], forces=np.zeros((0, 3)), normals=np.zeros((0, 3)),
                 density=np.zeros((0, 3)))
    uw = np.array([[0, 0, 0, 1.0, 2.0, 3.0], [0, 0, 0, -1.0, 0.5, 0.25]])
    r = np.array([[0.05, 0, 0], [2.0, 0, 0]])
    (ext, _, _), inside, rigid = gr.listener_gradient(empty, empty, body, r, ETA, [1, 1], [[0.4, 0, 0]] * 2, uw)
    assert inside.tolist() == [True, False]
    w = uw[1, 3:]
    assert np.array_equal(rigid[0, :9].reshape(3, 3),
                          np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]))  # the last body wins
    assert np.isnan(rigid[0, 9]) and ext[1, 9] == 0 and np.isfinite(np.asarray(ext[1], dtype=np.float64)).all()
    # the rigid gradient is that of U + omega x dx
    dx = np.array([0.3, -0.2, 0.1])
    assert np.allclose(gr.rigid_gradient(w)[:9].reshape(3, 3) @ dx, np.cross(w, dx), rtol=0, atol=1e-15)


def test_listener_gradient_is_marshalled_as_declared(calls):
    s = _inputs(5)
    fl = capi.Flow(0)
    _drive(fl, calls, [c for c in _twin_calls(s) if c[0] not in ("step", "stats")])
    r = np.arange(12, dtype=np.float64).reshape(4, 3)
    n0 = len(calls)
    G, p = capi.listener_gradient(fl, r)
    (name, args), = calls[n0:]
    assert name == "skb_flow_listener_gradient"
    assert args[1] == ("<f8", r.tobytes()) and args[2] == 4
    assert G.shape == (4, 3, 3) and p.shape == (4,)
    fl.close()
    mf = capi.MultiFlow(2)
    with pytest.raises(TypeError, match="capi.Flow"):
        capi.listener_gradient(mf, r)
    mf.close()

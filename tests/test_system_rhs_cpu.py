"""CPU tests of tests/system_rhs_reference.py, the restatement the device's system RHS (skb_flow_build_system_rhs) is
held to: closed forms in a uniform background flow, and every planted defect of RHS_DEFECTS missing the 1e-12 gate by
orders of magnitude.  The binding's argument checks need no GPU either."""
import numpy as np
import pytest

import system_rhs_reference as rr
from oracle import fiber_fd
from skellysim_b200 import capi
from test_fiber_rhs_cpu import ADV_POS, ADV_TENSION, U, advection_case

ETA, DT = 0.9, 1e-2


def small_case(seed, n_fibers=6, n_shell=40, body_nodes=(20, 30)):
    """slightly curved fibers of 8..24 nodes, a periphery, bodies, point sources and a background flow"""
    rng = np.random.default_rng(seed)
    n_nodes = rng.choice((8, 16, 24), size=n_fibers)
    lengths = rng.uniform(0.6, 1.6, n_fibers)
    pos = []
    for n, L in zip(n_nodes, lengths):
        t = rng.normal(size=3)
        t /= np.linalg.norm(t)
        pos.append(rng.uniform(-2, 2, 3) + np.linspace(0, L, n)[:, None] * t
                   + 0.05 * np.sin(np.linspace(0, 3, n))[:, None] * rng.normal(size=3))
    fib = dict(pos=np.concatenate(pos), n_nodes=[int(n) for n in n_nodes], lengths=list(lengths))
    d = rng.normal(size=(n_shell, 3))
    d /= np.linalg.norm(d, axis=1)[:, None]
    shell = dict(pos=6.0 * d, normals=-d)
    centers = rng.uniform(-1.5, 1.5, (len(body_nodes), 3))
    bp, bn = [], []
    for c, n in zip(centers, body_nodes):
        e = rng.normal(size=(n, 3))
        e /= np.linalg.norm(e, axis=1)[:, None]
        bp.append(c + 0.4 * e)
        bn.append(e)
    bodies = dict(pos=np.concatenate(bp), normals=np.concatenate(bn), centers=centers, n_nodes=list(body_nodes))
    fparams = [dict(length_prev=L * rng.uniform(0.95, 1.05), bending_rigidity=rng.uniform(1e-3, 1e-2),
                    radius=0.0125, penalty_param=500.0, beta_tstep=1.0, minus_clamped=bool(f % 2),
                    plus_pinned=bool((f // 2) % 2)) for f, L in enumerate(lengths)]
    nf = fib["pos"].shape[0]
    kw = dict(f_ext=rng.uniform(-1, 1, (nf, 3)), ft=rng.uniform(-1, 1, (len(body_nodes), 6)),
              points=(rng.uniform(-1, 1, (3, 3)), rng.normal(size=(3, 3)), rng.normal(size=(3, 3))),
              background=([1, 0, 2], np.array([0.5, -0.25, 0.1]), np.array([0.1, 0.2, -0.3])),
              v_growth=rng.uniform(-1, 1, n_fibers), force_scale=rng.uniform(-2, 2, n_fibers))
    return fib, shell, bodies, fparams, kw


def test_uniform_background_alone():
    """only a uniform background U: the shell rows are -U, each body's rows [-U ... ; 0], the fiber block that of a
    fiber in the flow U"""
    fib, shell, bodies, fparams, _ = small_case(1)
    Uf = np.array([0.3, -0.7, 0.2])
    rhs, v = rr.system_rhs(fib, shell, bodies, fparams, ETA, DT, background=([0, 1, 2], np.zeros(3), Uf))
    assert np.array_equal(v, np.tile(Uf, (v.shape[0], 1)))
    nf, ns = fib["pos"].shape[0], shell["pos"].shape[0]
    _, s, b = (rhs[:4 * nf], rhs[4 * nf:4 * nf + 3 * ns], rhs[4 * nf + 3 * ns:])
    assert np.array_equal(s, -np.tile(Uf, ns))
    off = 0
    for n in bodies["n_nodes"]:
        assert np.array_equal(b[off:off + 3 * n], -np.tile(Uf, n))
        assert np.array_equal(b[off + 3 * n:off + 3 * n + 6], np.zeros(6))
        off += 3 * n + 6


@pytest.mark.parametrize("n", (8, 32, 64))
def test_straight_free_fiber_in_uniform_background_is_advected(n):
    """a straight, free, force-free fiber: A_ y = its block of the system RHS gives x + dt U and zero tension, within
    the bound of tests/test_fiber_rhs_cpu.py"""
    x, L, Uf = advection_case(n)
    fib = dict(pos=x, n_nodes=[n], lengths=[L])
    empty = dict(pos=np.zeros((0, 3)), normals=np.zeros((0, 3)), centers=np.zeros((0, 3)), n_nodes=[])
    fp = [dict(length_prev=L, bending_rigidity=2.5e-3, radius=0.0125, penalty_param=500.0, beta_tstep=1.0,
               minus_clamped=False, plus_pinned=False)]
    rhs, _ = rr.system_rhs(fib, empty, empty, fp, ETA, DT, background=([0, 1, 2], np.zeros(3), Uf))
    fo = fiber_fd.FiberOperators(x, L, eta=ETA, dt=DT)
    y = np.linalg.solve(fo.A, rhs)
    pos = y[:3 * n].reshape(3, n).T
    cond = np.linalg.cond(fo.A)
    assert np.abs(pos - (x + DT * Uf)).max() <= ADV_POS * cond * U * np.abs(x).max()
    assert np.abs(y[3 * n:]).max() <= ADV_TENSION * cond * U


@pytest.mark.parametrize("defect", rr.RHS_DEFECTS)
def test_each_planted_defect_misses_the_gate(defect):
    fib, shell, bodies, fparams, kw = small_case(2)
    good, _ = rr.system_rhs(fib, shell, bodies, fparams, ETA, DT, **kw)
    bad, _ = rr.system_rhs(fib, shell, bodies, fparams, ETA, DT, defect=defect, **kw)
    nf, ns = fib["pos"].shape[0], shell["pos"].shape[0]
    worst = 0.0
    for sl in (slice(0, 4 * nf), slice(4 * nf, 4 * nf + 3 * ns), slice(4 * nf + 3 * ns, None)):
        ref = good[sl]
        worst = max(worst, np.abs(bad[sl] - ref).max() / max(np.abs(ref).max(), 1e-300))
    assert worst > 1e-6, (defect, worst)


def test_without_any_force_or_source_the_flow_is_zero():
    fib, shell, bodies, fparams, kw = small_case(3)
    _, v = rr.system_rhs(fib, shell, bodies, fparams, ETA, DT)
    assert not np.any(v)
    _, v0 = rr.system_rhs(fib, shell, bodies, fparams, ETA, DT, ft=np.zeros((2, 6)))
    assert not np.any(v0)


def test_rhs_binding_argument_shapes():
    p, vg, fs, f, ft = capi._system_rhs_args(3, 24, 2, (1.0, 2.5e-3, 0.0125, 500.0, 1.0, 0, [0, 1, 0]), 0.5, None,
                                             np.zeros((24, 3)), np.zeros((2, 6)))
    assert p["plus_hinged"].tolist() == [0, 1, 0] and vg.tolist() == [0.5] * 3 and fs is None
    assert f.shape == (24, 3) and ft.shape == (2, 6)
    with pytest.raises(ValueError, match=r"\(2, 6\)"):
        capi._system_rhs_args(3, 24, 2, (1.0,) * 5 + (0, 0), None, None, None, np.zeros((3, 6)))
    with pytest.raises(ValueError, match=r"\(24, 3\)"):
        capi._system_rhs_args(3, 24, 2, (1.0,) * 5 + (0, 0), None, None, np.zeros((23, 3)), None)


def test_rhs_entry_points_refuse_null_handles():
    import ctypes as C
    L = capi.library()
    null = C.c_void_p()
    p = capi.fiber_params(1, 1.0, 1.0, 0.01, 500.0, 1.0, 0, 0)
    out = np.zeros(32)
    calls = [
        lambda: L.skb_flow_build_system_rhs(null, capi._params_ptr(p), None, None, None, None, 1e-2, 1.0,
                                            capi._p(out)),
        lambda: L.skb_flow_build_system_rhs_device(null, capi._params_ptr(p), None, None, None, None, None, 1e-2, 1.0,
                                                   None, None),
        lambda: L.skb_mflow_build_system_rhs(null, capi._params_ptr(p), None, None, None, None, 1e-2, 1.0,
                                             capi._p(out)),
        lambda: L.skb_mflow_set_point_sources(null, None, None, None, 0),
        lambda: L.skb_mflow_set_background(null, None, None, None),
    ]
    for call in calls:
        assert call() != 0
        assert b"NULL" in L.skb_last_error_string()

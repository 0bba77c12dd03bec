"""CPU tests of the fiber block of the RHS (skb_flow_build_fiber_rhs, include/skelly_b200_flow.h) and of its reference,
tests/fiber_rhs_reference.py::fiber_rhs, evaluated on oracle/fiber_fd.py::FiberOperators.

The device RHS is held entry by entry to |dev - ext| <= C_RHS u S: ext the oracle evaluated in np.longdouble on the same
float64 inputs, S the same computation on absolute values (FiberOperators(absolute=True)), u = 2^-53.  These tests show
the criterion attainable (the float64 oracle meets it) and sharp (each planted defect of fiber_rhs_reference.RHS_DEFECTS
fails it), on curved fibers with n = 8 .. 128 and all four boundary-condition combinations, length_ != length_prev,
nonzero v_growth and force_scale, and f_external unlike the motor force.  A physics check solves A_ y = RHS for a
straight, free, force-free fiber in a uniform flow U: y is the fiber advected by dt U, with zero tension.  The NULL-
handle refusals and the binding's argument checks need no GPU either."""
import ctypes as C

import numpy as np
import pytest

from fiber_rhs_reference import RHS_DEFECTS, fiber_rhs
from oracle import fiber_fd
from skellysim_b200 import capi

NODES = (8, 16, 24, 32, 48, 64, 96, 128)
ETA, DT = 0.9, 5e-3
U = 2.0 ** -53
C_RHS = 8.0


def rhs_case(seed, n):
    """one curved fiber per boundary-condition combination: (FiberOperators kwargs, rhs kwargs) of each"""
    rng = np.random.default_rng(seed)
    out = []
    for combo in range(4):
        L = rng.uniform(0.6, 1.6)
        s = np.linspace(0.0, L, n)
        k, tau = rng.uniform(0.3, 1.5), rng.uniform(-1.0, 1.0)
        a = np.hypot(k, tau)
        c = np.stack([k / a ** 2 * np.cos(a * s), k / a ** 2 * np.sin(a * s), tau / a * s], axis=1)
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        ops = dict(x=rng.uniform(-4, 4, 3) + c @ q.T, length=L, length_prev=L * rng.uniform(0.9, 1.1),
                   bending_rigidity=rng.uniform(1e-3, 1e-2), radius=rng.uniform(5e-3, 2e-2), eta=ETA, dt=DT,
                   penalty_param=rng.uniform(100.0, 800.0), beta_tstep=rng.uniform(0.5, 1.5),
                   minus_clamped=bool(combo & 1), plus_pinned=bool(combo >> 1))
        rhs = dict(v=rng.uniform(-1, 1, (n, 3)), f_external=rng.uniform(-1, 1, (n, 3)),
                   force_scale=rng.uniform(-2, 2), v_growth=rng.uniform(-1, 1))
        out.append((ops, rhs))
    return out


def ratio(got, ext, S):
    """max over the entries of |got - ext| / (u S); a structural zero (S = 0) counts 0 if exactly zero, inf if not"""
    d = np.abs(np.asarray(got, dtype=np.float64).astype(np.longdouble) - ext).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(S > 0, d / (U * S), np.where(d == 0, 0.0, np.inf))
    return float(np.max(r))


def references(ops, rhs, **kw):
    """(float64, long double, S) of one fiber's RHS"""
    return tuple(fiber_rhs(fiber_fd.FiberOperators(ops["x"], **{k: v for k, v in ops.items() if k != "x"}, **d),
                           **rhs, **kw) for d in ({}, dict(dtype=np.longdouble), dict(absolute=True)))


@pytest.fixture(scope="module")
def cases():
    return {n: rhs_case(100 + n, n) for n in NODES}


def test_rhs_criterion_holds_for_the_fp64_oracle(cases):
    assert np.finfo(np.longdouble).nmant >= 63
    worst = {}
    for n, fibers in cases.items():
        for ops, rhs in fibers:
            for drop in (None, "v", "f_external", "force_scale", "all"):
                r = dict(rhs)
                if drop == "all":
                    r = dict(v_growth=0.0)
                elif drop:
                    r.pop(drop)
                got, ext, S = references(ops, r)
                worst[n] = max(worst.get(n, 0.0), ratio(got, ext, S))
                assert worst[n] <= C_RHS, (n, drop, worst[n])
    print("\nfp64 oracle RHS |d|/(u S), worst per n:", {n: round(w, 2) for n, w in worst.items()})


@pytest.mark.parametrize("defect", RHS_DEFECTS)
def test_rhs_criterion_catches_planted_defects(cases, defect):
    smallest = np.inf
    for n, fibers in cases.items():
        for ops, rhs in fibers:
            if defect == "swap_bc" and ops["minus_clamped"] == ops["plus_pinned"]:
                continue                                   # swapping equal branches changes nothing
            _, ext, S = references(ops, rhs)
            bad = fiber_rhs(fiber_fd.FiberOperators(ops["x"], **{k: v for k, v in ops.items() if k != "x"}), **rhs,
                            defect=defect)
            r = ratio(bad, ext, S)
            smallest = min(smallest, r)
            assert r > C_RHS, (defect, n, ops["minus_clamped"], ops["plus_pinned"], r)
    print(f"\n{defect}: smallest |d|/(u S) {smallest:.3g}")


# The solve's error follows cond(A_) (8e4 .. 4e8 here, at dt = 1e-2).  Over three seeds of advection_case and every n,
# numpy's float64 solve reached 3.2 cond u max|x| in the positions (1.2e-14 .. 4.7e-11) and 54 cond u in the tension
# (9.8e-14 .. 4.5e-10); a wrong RHS errs by O(dt |U|) or more.
ADV_POS, ADV_TENSION = 16.0, 256.0


def advection_case(n, seed=0):
    rng = np.random.default_rng(seed + n)
    L = rng.uniform(0.5, 2.0)
    t = rng.normal(size=3)
    t /= np.linalg.norm(t)
    x = rng.uniform(-2, 2, 3) + np.linspace(0.0, L, n)[:, None] * t
    Uf = rng.uniform(-1, 1, 3)
    return x, L, Uf


@pytest.mark.parametrize("n", NODES)
def test_straight_fiber_in_uniform_flow_is_advected(n):
    # a straight, free (Force / Torque at both ends), force-free fiber moves with the flow: A_ y = RHS gives
    # x + dt U and zero tension
    dt = 1e-2
    x, L, Uf = advection_case(n)
    fo = fiber_fd.FiberOperators(x, L, eta=ETA, dt=dt)
    y = np.linalg.solve(fo.A, fiber_rhs(fo, v=np.tile(Uf, (n, 1))))
    pos = y[:3 * n].reshape(3, n).T
    e_pos, e_t = np.abs(pos - (x + dt * Uf)).max(), np.abs(y[3 * n:]).max()
    cond = np.linalg.cond(fo.A)
    print(f"\nn = {n}: cond {cond:.1e}, position error {e_pos:.1e}, tension error {e_t:.1e}")
    assert e_pos <= ADV_POS * cond * U * np.abs(x).max() and e_t <= ADV_TENSION * cond * U


def test_rhs_entry_points_refuse_null_handles():
    L = capi.library()
    null = C.c_void_p()
    p = capi.fiber_params(1, 1.0, 1.0, 0.01, 500.0, 1.0, 0, 0)
    out = np.zeros(32)
    calls = [
        lambda: L.skb_flow_build_fiber_rhs(null, capi._params_ptr(p), None, None, None, None, 1e-2, 1.0,
                                           capi._p(out)),
        lambda: L.skb_flow_build_fiber_rhs_device(null, capi._params_ptr(p), None, None, None, None, 1e-2, 1.0,
                                                  None, None),
        lambda: L.skb_mflow_build_fiber_rhs(null, capi._params_ptr(p), None, None, None, None, 1e-2, 1.0,
                                            capi._p(out)),
    ]
    for call in calls:
        assert call() != 0
        assert b"NULL" in L.skb_last_error_string()


def test_rhs_binding_argument_shapes():
    p, vg, fs, v, f = capi._fiber_rhs_args(3, 24, (1.0, 2.5e-3, 0.0125, 500.0, 1.0, 0, [0, 1, 0]), 0.5, None,
                                           np.zeros((24, 3)), None)
    assert p["plus_hinged"].tolist() == [0, 1, 0] and vg.tolist() == [0.5] * 3 and fs is None and f is None
    assert v.shape == (24, 3)
    with pytest.raises(ValueError, match="3 values"):
        capi._fiber_rhs_args(3, 24, (1.0,) * 5 + (0, 0), [1.0, 2.0], None, None, None)
    with pytest.raises(ValueError, match=r"\(24, 3\)"):
        capi._fiber_rhs_args(3, 24, (1.0,) * 5 + (0, 0), None, None, np.zeros((23, 3)), None)

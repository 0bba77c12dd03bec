"""GPU tests of the dynamic instability (include/skelly_b200_flow.h skb_flow_dynamic_instability,
skb_flow_set_nucleation_sites, skb_flow_step_flags; timestep.Stepper with dynamic_instability) against
tests/dynamic_instability_reference.py, bitwise."""
import contextlib

import numpy as np
import pytest

import dynamic_instability_reference as dr
import skellysim_b200 as skb
import step_reference as st
from skellysim_b200 import capi, timestep
from test_gpu_step import EMPTY, ETA, periphery, random_unit_quaternion, set_classes
from test_gpu_system_edges import sphere

pytestmark = pytest.mark.gpu


def unit_dirs(n):
    return sphere(n, 1.0)[0]


@contextlib.contextmanager
def body_system(n_fib, n, n_sites, n_bodies=1, n_bound=2, n_shell=60, body_nodes=100, seed=5, free_at=3.0):
    """fibers (n_bound bound at the first sites of body 0, the rest free), n_bodies spheres of radius 0.5 with n_sites
    sites each, a periphery; every set-up call a step needs"""
    import system_reference as sr
    rng = np.random.default_rng(seed)
    R = 0.5
    centers = np.array([[4.0 * b - 2.0 * (n_bodies - 1), 0.3, -0.2] for b in range(n_bodies)])
    quats = np.array([random_unit_quaternion(rng) for _ in range(n_bodies)])
    site_ref = np.concatenate([R * unit_dirs(n_sites) for _ in range(n_bodies)]) if n_bodies else EMPTY
    pos = []
    for f in range(n_fib):
        if f < n_bound:
            d = site_ref[f] / R
            Rq = st.rotation(quats[0])
            pos.append(centers[0] + Rq @ site_ref[f] + np.linspace(0, 0.8, n)[:, None] * (Rq @ d))
        else:
            t = rng.normal(size=3)
            t /= np.linalg.norm(t)
            c = rng.uniform(-free_at, free_at, 3)
            pos.append(c + np.linspace(0, 0.8, n)[:, None] * t)
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0]))
        fl.set_fibers(np.concatenate(pos) if pos else EMPTY, [n] * n_fib, [0.8] * n_fib)
        r, nrm, M, Minv = periphery(n_shell, 5)
        fl.set_periphery(r, nrm)
        dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, M)
        dn.set_matrix(skb.DENSE_M_INV, Minv)
        rb, nb_, w = sphere(body_nodes, R)
        ex, ey, ez = sr.singularity_vectors(rb, nb_, w)
        A = sr.body_operator(rb, nb_, np.zeros(3), w, ex, ey, ez)
        Ai = np.linalg.inv(A)
        fl.set_bodies(np.concatenate([rb] * n_bodies), np.concatenate([nb_] * n_bodies), np.zeros((n_bodies, 3)))
        fl.set_body_frames([body_nodes] * n_bodies, np.concatenate([rb] * n_bodies), np.concatenate([nb_] * n_bodies),
                           np.concatenate([w] * n_bodies), *(np.concatenate([v] * n_bodies) for v in (ex, ey, ez)),
                           [Ai] * n_bodies)
        fl.place_bodies(centers, quats)
        fl.set_nucleation_sites([n_sites] * n_bodies, site_ref)
        set_classes(fl, [n])
        fl.set_gmres(300)
        binding = np.full((n_fib, 2), -1, dtype=np.int32)
        binding[:n_bound, 0], binding[:n_bound, 1] = 0, np.arange(n_bound)
        yield fl, dn, dict(binding=binding, site_ref=site_ref, n_sites=[n_sites] * n_bodies, n=n)


def base_params(n_fib, lengths=0.8):
    p = capi.fiber_params(n_fib, lengths, 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)
    return p


DI = dict(n_nodes=16, v_growth=0.3, f_catastrophe=10.5, v_grow_collision_scale=0.5, f_catastrophe_collision_scale=2.0,
          nucleation_rate=10.0, radius=0.0125, min_length=0.25, bending_rigidity=2.5e-3)


def reference(fl, sysd, di, dt, seed, counter, params, binding, pinned, r_fib, n_nodes, lengths):
    c, q = fl.placement()
    return dr.dynamic_instability(di, dt, seed, counter, lengths, params, binding, pinned, sysd["n_sites"],
                                  sysd["site_ref"], c, q, n_nodes_in=n_nodes, r_fib=r_fib)


def test_c3_like_is_bitwise_the_restatement():
    n_fib, n, dt = 3000, 32, 0.01
    with body_system(n_fib, n, 200, n_bodies=2, n_bound=150, n_shell=500, body_nodes=200, free_at=8.0) as (fl, dn, s):
        set_classes(fl, [16])
        rng = np.random.default_rng(9)
        lengths = rng.uniform(0.6, 1.2, n_fib)
        r0 = fl.fibers()
        fl.set_fibers(r0, [n] * n_fib, lengths)
        binding = s["binding"].copy()
        binding[100:150, 0], binding[100:150, 1] = 1, np.arange(50)
        p = base_params(n_fib, rng.uniform(0.5, 1.0, n_fib))
        pinned = (rng.uniform(size=n_fib) < 0.2).astype(np.int32)
        ref = reference(fl, s, DI, dt, 77, 5, p, binding, pinned, r0, [n] * n_fib, lengths)
        out = fl.dynamic_instability(DI, dt, 77, 5, p, binding, pinned)
        r_new = fl.fibers()
    print(f"\nremoved {out['removed']}, nucleated {out['nucleated']}, mu {out['mu']:.2f}")
    assert 200 <= out["removed"] <= 400 and out["nucleated"] >= 10
    for k in ("removed", "nucleated", "grown", "mu"):
        assert out[k] == ref[k], k
    assert out["params"].tobytes() == ref["params"].tobytes()
    assert np.array_equal(out["binding"], ref["binding"]) and np.array_equal(out["origin"], ref["origin"])
    assert np.array_equal(out["v_growth"], ref["v_growth"]) and np.array_equal(out["lengths"], ref["lengths"])
    assert np.array_equal(out["n_nodes"], ref["n_nodes"])
    assert np.array_equal(r_new, ref["positions"])


def step_args(out, s):
    body = out["binding"][:, 0]
    off = np.concatenate([[0], np.cumsum(s["n_sites"])])
    site_ref = s["site_ref"][np.where(body >= 0, off[np.maximum(body, 0)] + out["binding"][:, 1], 0)]
    p = out["params"]
    return (tuple(p[k] for k in capi.FIBER_PARAMS_DTYPE.names),
            dict(fiber_body=body, site_ref=site_ref, v_growth=out["v_growth"], tol=1e-12, num_blocks=200,
                 max_iters=400, body_forces_torques=np.array([[0.2, -0.1, 0.3, 0.3, -0.5, 0.4]])))


@pytest.mark.parametrize("shaped", [False, True])
def test_the_next_step_is_the_step_of_a_fresh_flow(shaped):
    dt = 0.02
    di = dict(DI, f_catastrophe=5.0, nucleation_rate=8.0)  # mu = 0.02 x 8 x 38 sites: about 6
    shape = dict(kind=capi.PERIPHERY_ELLIPSOID, a=12.0, b=11.0, c=13.0, f_0=20.0, l_0=0.5)
    with body_system(6, 16, 40) as (fl, dn, s):
        if shaped:
            fl.set_periphery_shape(**shape, fiber_minus_clamped=[1, 1, 0, 0, 0, 0])
        p = base_params(6)
        p["minus_clamped"][:2] = 1
        out = fl.dynamic_instability(di, dt, 3, 0, p, s["binding"], np.zeros(6, dtype=np.int32))
        assert out["nucleated"] > 0
        r, nn, L = fl.fibers(), out["n_nodes"], out["lengths"]
        params, kw = step_args(out, s)
        x, tension, info = fl.step(*params, dt, ETA, dense=dn, **kw)
        flags = fl._shape["fiber_minus_clamped"] if shaped else None
    with body_system(6, 16, 40) as (fresh, dn2, _):
        fresh.set_fibers(r, nn, L)
        if shaped:
            fresh.set_periphery_shape(**shape, fiber_minus_clamped=flags)
        fresh.set_gmres(300)
        x2, tension2, info2 = fresh.step(*params, dt, ETA, dense=dn2, **kw)
    assert np.array_equal(x, x2) and np.array_equal(tension, tension2)
    assert info == info2 or (np.isnan(info["fiber_error"]) and np.isnan(info2["fiber_error"]))


def test_all_fibers_removed_then_the_step_runs():
    with body_system(4, 16, 10) as (fl, dn, s):
        out = fl.dynamic_instability(dict(DI, f_catastrophe=1e9, nucleation_rate=0.0), 0.02, 1, 0, base_params(4),
                                     s["binding"], np.zeros(4, dtype=np.int32))
        assert out["removed"] == 4 and out["nucleated"] == 0 and fl.n_fib == 0
        _, _, info = fl.step([], 0, 1, 1, 1, 0, 0, 0.02, ETA, dense=dn, tol=1e-12, num_blocks=200, max_iters=400,
                             body_forces_torques=np.array([[0.2, -0.1, 0.3, 0.3, -0.5, 0.4]]))
        assert info["converged"] and info["worst_fiber"] == -1


def test_refusals_leave_the_fibers_untouched_and_a_group_member_is_refused():
    with body_system(4, 16, 10) as (fl, dn, s):
        r0 = fl.fibers()
        p, b, pin = base_params(4), s["binding"], np.zeros(4, dtype=np.int32)

        def refused(di=DI, dt=0.02, binding=b, pinned=pin):
            before = capi.launch_count()
            with pytest.raises(skb.SkbError, match="error 1:"):
                fl.dynamic_instability(di, dt, 1, 0, p, binding, pinned)
            assert capi.launch_count() == before and np.array_equal(fl.fibers(), r0) and fl.n_fib == 64

        refused(dt=0.0)
        refused(dt=float("nan"))
        refused(di=dict(DI, f_catastrophe=-1.0))
        refused(di=dict(DI, nucleation_rate=float("inf")))
        refused(di=dict(DI, min_length=0.0))
        refused(di=dict(DI, n_nodes=7))
        refused(di=dict(DI, n_nodes=24))  # no class
        bad = b.copy()
        bad[0] = (0, 10)
        refused(binding=bad)
        bad[0] = (1, 0)
        refused(binding=bad)
        refused(pinned=np.full(4, 2, dtype=np.int32))
        with pytest.raises(skb.SkbError, match="error 1:"):
            fl.set_nucleation_sites([2], np.zeros((2, 3)))
    with body_system(2, 16, 10) as (fl, dn, s):
        fl.set_bodies(*sphere(50, 0.5)[:2], np.zeros((1, 3)))  # new bodies: no sites for them yet, not placed
        with pytest.raises(skb.SkbError, match="error 1:"):
            fl.dynamic_instability(DI, 0.02, 1, 0, base_params(2), s["binding"], np.zeros(2, dtype=np.int32))
    with skb.Flow(0) as fl:
        fl.set_fibers(np.zeros((16, 3)) + np.linspace(0, 1, 16)[:, None], [16], [1.0])
        fl.set_periphery(EMPTY, EMPTY)
        fl.set_bodies(EMPTY, EMPTY, EMPTY)
        set_classes(fl, [16])
        fl.group_init(0, 2)
        with pytest.raises(skb.SkbError, match="error 1:.*group member"):
            fl.dynamic_instability(DI, 0.02, 1, 0, base_params(1), [[-1, -1]], [0])


def run_once(seed):
    """timestep.run with the model on, dt fixed but for the halving of the two steps the collision callable rejects
    (about 55 steps); every restore checked against the backup"""
    dt = 0.01
    di = dict(DI, f_catastrophe=3.0, nucleation_rate=5.0)
    calls = []
    with body_system(6, 16, 40) as (fl, dn, s):
        class Checked(timestep.Stepper):
            def backup(self):
                super().backup()
                self._want = (self.flow.fibers(), self.flow._fiber_off.copy(), self.flow._lengths.copy(),
                              tuple(a.copy() for a in self.params), self.binding.copy())

            def restore(self):
                super().restore()
                got = (self.flow.fibers(), self.flow._fiber_off, self.flow._lengths, self.params, self.binding)
                w = self._want
                assert all(np.array_equal(a, b) for a, b in zip(got[:3], w[:3]))
                assert all(np.array_equal(a, b) for a, b in zip(got[3], w[3])) and np.array_equal(got[4], w[4])

        stp = Checked(fl, dn, (0.8, 2.5e-3, 0.0125, 500.0, 1.0, np.array([1, 1, 0, 0, 0, 0]), 0), ETA,
                      fiber_body=s["binding"][:, 0], fiber_site=s["binding"][:, 1], tol=1e-10, num_blocks=200,
                      max_iters=400, dynamic_instability=di, seed=seed)

        def collided(r, c):
            calls.append(len(r))
            return len(calls) in (7, 15)

        t, dt_end, log = timestep.run(stp, 20 * dt, dt, dt_min=1e-4, dt_max=dt, beta_up=1.0, beta_down=1.0,
                                      fiber_error_tol=1e3, collided=collided)
        return log, fl.fibers(), stp.counter


def test_a_full_run_reproduces_and_restores_rejected_steps():
    log, r, counter = run_once(42)
    assert sum(1 for e in log if not e[2]) == 2 and len(log) >= 30 and counter == len(log)
    log2, r2, _ = run_once(42)
    assert log == log2 and np.array_equal(r, r2)

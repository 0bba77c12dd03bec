"""GPU tests of one timestep of the whole system (include/skelly_b200_flow.h skb_flow_step, skb_flow_fiber_error,
skb_flow_get_placement; skellysim_b200.timestep), against tests/step_reference.py.

FIBER ERROR BOUND: per fiber, |device - long double restatement| <= K u max_i S_i, with S_i step_reference.fiber_error's
scale and K = m + 10, m the widest non-zero row range of a column of D_1_0 (the longest sum, its products and the scale
2/L: m + 1 roundings per component; the squares, their sum and the root: 4; the difference with 1: 1; 4 spare)."""
import contextlib

import numpy as np
import pytest

import skellysim_b200 as skb
import step_reference as st
from oracle.fiber_fd import compute_matrices
from skellysim_b200 import capi, timestep
from test_gpu_system_edges import sphere

pytestmark = pytest.mark.gpu
ETA, DT = 0.9, 1e-3
U = 2.0 ** -53
EMPTY = np.zeros((0, 3))


def straight_fibers(n_fibers, n, seed):
    rng = np.random.default_rng(seed)
    pos, lengths = [], []
    for f in range(n_fibers):
        t = rng.normal(size=3)
        t /= np.linalg.norm(t)
        L = rng.uniform(0.6, 1.2)
        pos.append(np.array([3.0 * f, 0.0, 0.0]) + np.linspace(0.0, L, n)[:, None] * t)
        lengths.append(L)
    return pos, np.array(lengths)


def params_of(lengths, clamped=0):
    return (np.asarray(lengths), 2.5e-3, 0.0125, 500.0, 1.0, clamped, 0)


def set_classes(fl, nodes):
    for n in sorted(set(nodes)):
        m = compute_matrices(n)
        fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])


def periphery(n_shell, seed, nan=False):
    r, nrm, _ = sphere(n_shell, 12.0)
    rng = np.random.default_rng(seed)
    M = np.eye(3 * n_shell) + 0.1 * rng.normal(size=(3 * n_shell, 3 * n_shell)) / np.sqrt(3 * n_shell)
    Minv = np.linalg.inv(M)
    if nan:
        Minv[5, 7] = np.nan
    return r, -nrm, M, Minv


@contextlib.contextmanager
def fiber_flow(pos, lengths, n_shell=0, background=(0.3, -0.2, 0.5), nan=False, gmres=True):
    """free fibers (and a periphery) in a uniform background flow, every set-up call the step needs"""
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = None
        fl.set_fibers(np.concatenate(pos) if pos else EMPTY, [len(p) for p in pos], lengths)
        if n_shell:
            r, nrm, M, Minv = periphery(n_shell, 5, nan)
            fl.set_periphery(r, nrm)
            dn = stack.enter_context(skb.Dense(device_ids=[0]))
            dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, M)
            dn.set_matrix(skb.DENSE_M_INV, Minv)
        else:
            fl.set_periphery(EMPTY, EMPTY)
        fl.set_bodies(EMPTY, EMPTY, EMPTY)
        set_classes(fl, [len(p) for p in pos])
        fl.set_body_operators([], [], EMPTY, EMPTY, EMPTY)
        fl.set_background([0, 1, 2], np.zeros(3), np.array(background))
        if gmres:
            fl.set_gmres(300)
        yield fl, dn


def test_fiber_error_matches_the_long_double_restatement():
    rng = np.random.default_rng(11)
    nodes = [8, 16, 32, 64, 128, 24, 128, 8]
    pos, lengths = [], []
    for f, n in enumerate(nodes):
        L = rng.uniform(0.5, 2.0)
        s = np.linspace(0.0, L, n)
        k = rng.uniform(0.2, 2.0)  # a helix-like arc, stretched a little
        pos.append(np.stack([np.cos(k * s) / k, np.sin(k * s) / k, 0.3 * s], axis=1) * rng.uniform(0.9, 1.1)
                   + rng.normal(size=3) * 5)
        lengths.append(L)
    with skb.Flow(0) as fl:
        fl.set_fibers(np.concatenate(pos), nodes, lengths)
        for n in sorted(set(nodes)):
            m = compute_matrices(n)
            fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        before = capi.launch_count()
        e_max, per = fl.fiber_error()
        assert capi.launch_count() == before + 1
    worst = 0.0
    for f, n in enumerate(nodes):
        D = compute_matrices(n)["D_1_0"]
        m = max(int(np.ptp(np.nonzero(D[:, i])[0])) + 1 for i in range(n))
        e_ld, S = st.fiber_error(pos[f], lengths[f], D, dtype=np.longdouble)
        ref = float(e_ld.max())
        ratio = abs(per[f] - ref) / ((m + 10) * U * S.max())
        worst = max(worst, ratio)
    print(f"\nfiber error: worst ratio to the bound {worst:.3f}; max {e_max:.3e}")
    assert worst <= 1.0
    assert e_max == per.max()


def composed(fl, dn, params, n_iters=1000, tol=1e-12):
    """the existing calls a caller composes: links, the build, the RHS, the solve"""
    fl.set_fiber_links(None)
    fl.build_fiber_operators(*params, DT, ETA)
    b = fl.build_system_rhs(*params, DT, ETA)
    x, info, _ = fl.solve_system(b, ETA, dense=dn, tol=tol, max_iters=n_iters)
    return x, info


@pytest.mark.parametrize("n_shell", [0, 200])
def test_the_step_is_the_composition_and_its_restatement(n_shell):
    pos, lengths = straight_fibers(5, 16, 66)
    p = params_of(lengths)
    with fiber_flow(pos, lengths, n_shell) as (fl, dn):
        x_ref, i_ref = composed(fl, dn, p)
    with fiber_flow(pos, lengths, n_shell) as (fl, dn):
        x, tension, info = fl.step(*p, DT, ETA, dense=dn, tol=1e-12)
        r_new = fl.fibers()
        e_now, _ = fl.fiber_error()
    assert np.array_equal(x, x_ref), np.abs(x - x_ref).max()
    assert {k: info[k] for k in i_ref} == i_ref
    new = st.fiber_step(x[:4 * 16 * 5], [16] * 5)
    assert np.array_equal(r_new, np.concatenate([q for q, _ in new]))
    assert np.array_equal(tension, np.concatenate([t for _, t in new]))
    errs = [st.fiber_error(q, L, compute_matrices(16)["D_1_0"])[0].max() for (q, _), L in zip(new, lengths)]
    assert info["fiber_error"] == e_now and info["worst_fiber"] >= 0
    assert abs(info["fiber_error"] - max(errs)) <= 1e-13


def test_free_fibers_advect_with_zero_tension_over_five_steps_and_steps_reproduce():
    pos, lengths = straight_fibers(4, 16, 67)
    Uf = np.array([0.3, -0.2, 0.5])
    p = params_of(lengths)
    with fiber_flow(pos, lengths, background=Uf) as (fl, dn):
        st_ = timestep.Stepper(fl, dn, p, ETA, tol=1e-14)
        for k in range(1, 6):
            st_.backup()
            info = st_.step(DT)
            r1 = fl.fibers()
            st_.restore()
            info2 = st_.step(DT)
            assert np.array_equal(fl.fibers(), r1) and info == info2  # two steps from one state agree bit for bit
            assert info["converged"]
            err = np.abs(fl.fibers() - (np.concatenate(pos) + k * DT * Uf)).max()
            assert err <= 1e-12, (k, err)
            # a position error of 1e-12 moves xs by at most 1e-12 (2/L) max_i sum_j |D_ji| (< 4 (n - 1) / L here)
            assert info["fiber_error"] <= 1e-12 * 4 * 15 / lengths.min() + 1e-14
        x, tension, _ = fl.step(*p, DT, ETA, tol=1e-14)
    assert np.abs(tension).max() <= 1e-9


def sphere_flow(stack, n, R, fibers=None):
    import system_reference as sr
    r, nrm, w = sphere(n, R)
    ex, ey, ez = sr.singularity_vectors(r, nrm, w)
    A = sr.body_operator(r, nrm, np.zeros(3), w, ex, ey, ez)
    fl = stack.enter_context(skb.Flow(0))
    pos, nodes, lengths = fibers if fibers else ([], [], [])
    fl.set_fibers(np.concatenate(pos) if pos else EMPTY, nodes, lengths)
    fl.set_periphery(EMPTY, EMPTY)
    fl.set_bodies(r, nrm, np.zeros((1, 3)))
    set_classes(fl, nodes)
    fl.set_body_frames([n], r, nrm, w, ex, ey, ez, [np.linalg.inv(A)])
    fl.place_bodies(np.zeros((1, 3)), np.array([[1.0, 0.0, 0.0, 0.0]]))
    fl.set_gmres(200)
    return fl


def test_a_sphere_turns_by_its_rotlet_and_moves_by_stokes_law():
    n, R, eta, k, dt = 400, 0.5, 0.7, 4, 0.05
    L = np.array([0.2, 0.5, -0.4])
    ft = np.concatenate([np.zeros(3), L])[None]
    with contextlib.ExitStack() as stack:
        fl = sphere_flow(stack, n, R)
        for _ in range(k):
            _, _, info = fl.step(1.0, 2.5e-3, 0.0125, 500.0, 1.0, 0, 0, dt, eta, body_forces_torques=ft, tol=1e-13,
                                 num_blocks=200)
            assert info["converged"] and info["fiber_error"] == 0 and info["worst_fiber"] == -1
        c, q = fl.placement()
    W = L / (8 * np.pi * eta * R ** 3)
    from test_step_cpu import rodrigues
    want = rodrigues(k * dt * W)
    err = np.abs(st.rotation(q[0]) - want).max() / (k * dt * np.linalg.norm(W))
    print(f"\nrotation error {err:.2e}, |c| {np.abs(c).max():.1e}")
    assert err <= 1e-12 and np.abs(c).max() <= 1e-12
    R, eta, F = 1.0, 1.0, np.array([0.3, -0.7, 0.2])
    with contextlib.ExitStack() as stack:
        fl = sphere_flow(stack, n, R)
        for _ in range(k):
            fl.step(1.0, 2.5e-3, 0.0125, 500.0, 1.0, 0, 0, dt, eta,
                    body_forces_torques=np.concatenate([F, np.zeros(3)])[None], tol=1e-13, num_blocks=200)
        c, q = fl.placement()
    want = k * dt * F / (6 * np.pi * eta * R)
    e = np.linalg.norm(c[0] - want) / np.linalg.norm(want)
    print(f"translation error {e:.2e}")
    # the lattice's discretisation also turns it a little under a pure force (|w| ~ 1e-6 here)
    assert e <= 2 * 3.1e-5 and np.abs(q[0] - [1.0, 0.0, 0.0, 0.0]).max() <= 1e-6


def test_bound_fibers_stay_at_their_rotated_sites():
    n, R, dt = 400, 0.5, 0.02
    rng = np.random.default_rng(12)
    dirs = rng.normal(size=(3, 3))
    dirs /= np.linalg.norm(dirs, axis=1)[:, None]
    nf, m = 3, 16
    pos = [R * 1.0 * d + np.linspace(0, 0.8, m)[:, None] * d for d in dirs]
    site_ref = R * dirs
    ft = np.array([[0.0, 0.0, 0.0, 0.3, -0.2, 0.4]])
    with contextlib.ExitStack() as stack:
        fl = sphere_flow(stack, n, R, fibers=(pos, [m] * nf, [0.8] * nf))
        for _ in range(3):
            _, _, info = fl.step(np.full(nf, 0.8), 2.5e-3, 0.0125, 500.0, 1.0, 1, 0, dt, ETA, body_forces_torques=ft,
                                 fiber_body=[0] * nf, site_ref=site_ref, tol=1e-10, num_blocks=200, max_iters=400)
            c, q = fl.placement()
            r = fl.fibers().reshape(nf, m, 3)
            for f in range(nf):
                s = st.site(c[0], q[0], site_ref[f])
                assert np.all(np.abs(r[f, 0] - s) <= 2 * U * (np.abs(r[f, 0]) + np.abs(s)) + 1e-15), (f, r[f, 0], s)
            assert np.isfinite(info["fiber_error"])
        assert abs(np.dot(q[0], q[0]) - 1) <= 4 * U and q[0][0] < 1.0  # it turned


def test_refusals_change_nothing_and_launch_nothing():
    pos, lengths = straight_fibers(3, 16, 68)
    p = params_of(lengths)
    with fiber_flow(pos, lengths, gmres=False) as (fl, dn):
        r0 = fl.fibers()

        def refused(**kw):
            before = capi.launch_count()
            args = dict(dict(dt=DT, fiber_body=None), **kw)
            with pytest.raises(skb.SkbError, match="error 1:"):
                fl.step(*p, args.pop("dt"), ETA, **args)
            assert capi.launch_count() == before and np.array_equal(fl.fibers(), r0)

        refused()  # no set_gmres
        fl.set_gmres(50)
        refused(dt=0.0)
        refused(dt=float("nan"))
        refused(dt=float("inf"))
        refused(fiber_body=[0, -1, -1])  # no bodies
        refused(fiber_body=[-2, -1, -1])
        refused(num_blocks=51)
        refused(f_external=np.full((48, 3), np.nan))
    # bodies not placed from frames
    r, nrm, w = sphere(50, 1.0)
    with skb.Flow(0) as fl:
        fl.set_fibers(EMPTY, [], [])
        fl.set_periphery(EMPTY, EMPTY)
        fl.set_bodies(r, nrm, np.zeros((1, 3)))
        fl.set_body_operators([50], w, r, r, r, [np.eye(156)])
        fl.set_gmres(10)
        before = capi.launch_count()
        with pytest.raises(skb.SkbError, match="error 1:.*frames"):
            fl.step([], 0, 1, 1, 1, 0, 0, DT, ETA)
        with pytest.raises(skb.SkbError, match="error 1:"):
            fl.placement()
        assert capi.launch_count() == before


def test_a_non_finite_solution_is_not_installed():
    pos, lengths = straight_fibers(3, 16, 69)
    p = params_of(lengths)
    with fiber_flow(pos, lengths, n_shell=100, nan=True) as (fl, dn):
        r0 = fl.fibers()
        _, _, info = fl.step(*p, DT, ETA, dense=dn, max_iters=5)
        assert np.isnan(info["fiber_error"]) and info["worst_fiber"] == -1
        assert np.array_equal(fl.fibers(), r0)


def test_the_empty_system_steps_without_a_launch():
    with skb.Flow(0) as fl:
        fl.set_fibers(EMPTY, [], [])
        fl.set_periphery(EMPTY, EMPTY)
        fl.set_bodies(EMPTY, EMPTY, EMPTY)
        before = capi.launch_count()
        x, t, info = fl.step([], 0, 1, 1, 1, 0, 0, DT, ETA)
        assert capi.launch_count() == before and x.size == 0 and info["converged"] == 1
        assert info["fiber_error"] == 0 and info["worst_fiber"] == -1


def test_run_accepts_every_free_fiber_step_and_grows_dt_to_dt_max():
    pos, lengths = straight_fibers(3, 16, 70)
    with fiber_flow(pos, lengths) as (fl, dn):
        s = timestep.Stepper(fl, dn, params_of(lengths), ETA, tol=1e-12)
        t, dt, log = timestep.run(s, 0.02, 1e-3, dt_min=1e-6, dt_max=4e-3, beta_up=1.5, fiber_error_tol=0.1)
    assert all(acc for _, _, acc, _ in log)
    assert max(d for _, d, _, _ in log) == 4e-3 and dt == 4e-3
    assert t >= 0.02 and t - log[-1][1] < 0.02


# ---- a body with bound fibers, turning off its axis; the same over skb_mflow ------------------------------------------


def random_unit_quaternion(rng):
    q = rng.normal(size=4)
    return q / np.linalg.norm(q)


def step_case(name, seed=21):
    """FP: free fibers in a periphery; FPB: a 100-node sphere placed at a non-identity orientation, two fibers bound to
    it and one free, in a periphery, under a force and a torque off any axis of the orientation; B: the body alone"""
    rng = np.random.default_rng(seed)
    case = dict(fibers=[], lengths=[], body=None, n_shell=0, fiber_body=None, site_ref=None, clamped=[], ft=None)
    if name in ("FP", "FPB"):
        case["n_shell"] = 60
    if name == "FP":
        pos, lengths = straight_fibers(3, 16, seed)
        case.update(fibers=pos, lengths=list(lengths), clamped=[0, 0, 0])
    if name in ("FPB", "B"):
        R = 0.5
        q0 = random_unit_quaternion(rng)
        c0 = np.array([0.2, -0.1, 0.3])
        case.update(body=dict(n=100, R=R, c0=c0, q0=q0), ft=np.array([[0.2, -0.1, 0.3, 0.3, -0.5, 0.4]]))
    if name == "FPB":
        Rq = st.rotation(case["body"]["q0"])
        dirs = rng.normal(size=(2, 3))
        dirs /= np.linalg.norm(dirs, axis=1)[:, None]
        site_ref = np.concatenate([0.5 * dirs, np.zeros((1, 3))])
        pos = [case["body"]["c0"] + Rq @ (0.5 * d) + np.linspace(0, 0.8, 16)[:, None] * (Rq @ d) for d in dirs]
        pos.append(np.array([3.0, 0.0, 0.0]) + np.linspace(0, 0.8, 16)[:, None] * np.array([0.0, 0.6, 0.8]))
        case.update(fibers=pos, lengths=[0.8] * 3, fiber_body=[0, 0, -1], site_ref=site_ref, clamped=[1, 1, 0])
    return case


def set_up(fl, dn, case):
    """every set-up call the step needs, on a Flow (dn its Dense) or a MultiFlow (dn None)"""
    import system_reference as sr
    pos = case["fibers"]
    fl.set_fibers(np.concatenate(pos) if pos else EMPTY, [len(p) for p in pos], case["lengths"])
    if case["n_shell"]:
        r, nrm, M, Minv = periphery(case["n_shell"], 5, case.get("nan", False))
        fl.set_periphery(r, nrm)
        for op, A in ((skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, M), (skb.DENSE_M_INV, Minv)):
            dn.set_matrix(op, A) if dn is not None else fl.set_dense(op, A)
    else:
        fl.set_periphery(EMPTY, EMPTY)
    b = case["body"]
    if b:
        r, nrm, w = sphere(b["n"], b["R"])
        ex, ey, ez = sr.singularity_vectors(r, nrm, w)
        A = sr.body_operator(r, nrm, np.zeros(3), w, ex, ey, ez)
        fl.set_bodies(r, nrm, np.zeros((1, 3)))
        fl.set_body_frames([b["n"]], r, nrm, w, ex, ey, ez, [np.linalg.inv(A)])
        fl.place_bodies(b["c0"][None], b["q0"][None])
    else:
        fl.set_bodies(EMPTY, EMPTY, EMPTY)
        fl.set_body_operators([], [], EMPTY, EMPTY, EMPTY)
    if pos:
        set_classes(fl, [len(p) for p in pos])
    fl.set_background([0, 1, 2], np.zeros(3), np.array([0.3, -0.2, 0.5]))
    fl.set_gmres(300)


def case_params(case):
    return (np.asarray(case["lengths"]), 2.5e-3, 0.0125, 500.0, 1.0, np.asarray(case["clamped"], dtype=np.int32), 0)


def step_of(fl, dn, case, dt=0.02):
    return fl.step(*case_params(case), dt, ETA, dense=dn, body_forces_torques=case["ft"],
                   fiber_body=case["fiber_body"], site_ref=case["site_ref"], tol=1e-12, num_blocks=200,
                   max_iters=400)


def check_against_restatement(fl, case, x, tension, c_prev, q_prev, dt=0.02):
    """the flow's new positions, tensions and placement are the restatement of the step applied to its own x"""
    nodes = [len(p) for p in case["fibers"]]
    n_fib = sum(nodes)
    new = st.fiber_step(x[:4 * n_fib], nodes)
    if case["body"]:
        b0 = 4 * n_fib + 3 * case["n_shell"] + 3 * case["body"]["n"]
        c_new, q_new = st.body_step(c_prev[0], q_prev[0], x[b0:b0 + 3], x[b0 + 3:b0 + 6], dt)
        c, q = fl.placement()
        assert np.abs(c[0] - c_new).max() <= 4 * U * np.abs(c_new).max(), (c[0], c_new)
        assert np.abs(q[0] - q_new).max() <= 4 * U, (q[0], q_new)
        _, q_right = st.body_step(c_prev[0], q_prev[0], x[b0:b0 + 3], x[b0 + 3:b0 + 6], dt, right=True)
        assert np.abs(q_right - q_new).max() > 1e-9  # the test tells q * q_phi from q_phi * q here
    r = fl.fibers()
    off = 0
    for f, (p, _) in enumerate(new):
        got = r[off:off + len(p)]
        off += len(p)
        if case["fiber_body"] is not None and case["fiber_body"][f] >= 0:
            s = st.site(c_new, q_new, case["site_ref"][f])
            want = st.repin(p, s)
            assert np.all(np.abs(got - want) <= 8 * U * (np.abs(p) + np.abs(s))), f
            assert np.all(np.abs(got[0] - s) <= 8 * U * (np.abs(p[0]) + np.abs(s))), f
        else:
            assert np.array_equal(got, p), f
    assert np.array_equal(tension, np.concatenate([t for _, t in new]) if new else np.zeros(0))


def test_bound_fibers_on_a_body_turning_off_its_axis_step_as_the_composition_and_the_restatement():
    case = step_case("FPB")
    p = case_params(case)
    with fiber_flow([], [], gmres=False) as (twin, _), skb.Dense(device_ids=[0]) as dn2:
        set_up(twin, dn2, case)
        c, q = twin.placement()
        sites = np.array([st.site(c[0], q[0], s) for s in case["site_ref"]])
        twin.set_fiber_links(case["fiber_body"], sites, 2.5e-3)
        twin.build_fiber_operators(*p, 0.02, ETA)
        b = twin.build_system_rhs(*p, 0.02, ETA, body_forces_torques=case["ft"])
        x_ref, i_ref, _ = twin.solve_system(b, ETA, dense=dn2, tol=1e-12, num_blocks=200, max_iters=400)
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0]))
        set_up(fl, dn, case)
        for k in range(3):
            c, q = fl.placement()
            x, tension, info = step_of(fl, dn, case)
            if k == 0:
                assert np.array_equal(x, x_ref) and {key: info[key] for key in i_ref} == i_ref
            assert np.isfinite(info["fiber_error"]) and info["worst_fiber"] >= 0
            check_against_restatement(fl, case, x, tension, c, q)


def mflow_lists():
    n = capi.device_count()
    return [[0], [0, 0], [0, 0, 0]] + [list(range(k)) for k in (2, 3) if n >= k]


@pytest.mark.parametrize("name", ["FP", "FPB", "B"])
def test_mflow_steps_as_the_single_device(name):
    """[0] is bitwise skb_flow_step; more members (one owning no fiber, or nothing of a block) solve to the single
    device's solution within the solve's tolerance, and their new geometry is the restatement of their own solution"""
    case = step_case(name)
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0])) if case["n_shell"] else None
        set_up(fl, dn, case)
        single = []
        for _ in range(2):
            x, t, info = step_of(fl, dn, case)
            single.append((x, t, info, fl.fibers(), fl.placement() if case["body"] else None))
    for devs in mflow_lists():
        with skb.MultiFlow(devs) as mf:
            set_up(mf, None, case)
            for k in range(2):
                c, q = mf.placement() if case["body"] else (None, None)
                x, t, info = step_of(mf, None, case)
                xs, ts, infos, rs, pls = single[k]
                if devs == [0]:
                    assert np.array_equal(x, xs) and np.array_equal(t, ts) and info == infos
                    assert np.array_equal(mf.fibers(), rs)
                    if case["body"]:
                        assert all(np.array_equal(a, b) for a, b in zip(mf.placement(), pls))
                else:
                    assert info["converged"] and np.abs(x - xs).max() <= 1e-9 * np.abs(xs).max(), devs
                    check_against_restatement(mf, case, x, t, c, q)
                    assert abs(info["fiber_error"] - infos["fiber_error"]) <= 1e-9


def test_a_non_finite_solution_with_a_body_installs_nothing():
    case = dict(step_case("FPB"), nan=True)
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0]))
        set_up(fl, dn, case)
        r0, (c0, q0) = fl.fibers(), fl.placement()
        x, _, info = fl.step(*case_params(case), 0.02, ETA, dense=dn, body_forces_torques=case["ft"],
                             fiber_body=case["fiber_body"], site_ref=case["site_ref"], max_iters=5)
        assert np.isnan(info["fiber_error"]) and info["worst_fiber"] == -1 and not np.isfinite(x).all()
        c1, q1 = fl.placement()
        assert np.array_equal(fl.fibers(), r0) and np.array_equal(c0, c1) and np.array_equal(q0, q1)


def test_refusals_with_a_body_leave_fibers_and_placement_untouched():
    refusals_with_a_body(None)


def test_refusals_with_a_body_over_three_members_leave_fibers_and_placement_untouched():
    """the members own one fiber each, so that fiber_body=[0, 1, -1] is a refusal only member 1's fiber shows"""
    refusals_with_a_body([0, 0, 0])


def refusals_with_a_body(devs):
    """on a Flow (devs None) or over skb_mflow on devs: a refused step launches nothing and changes nothing, and the
    next step is bitwise the step of a twin that saw no refusal (over skb_mflow that step also fails if any member's
    flag wait timed out)"""
    case = step_case("FPB")

    def stepping(stack):
        if devs is None:
            fl, dn = stack.enter_context(skb.Flow(0)), stack.enter_context(skb.Dense(device_ids=[0]))
        else:
            fl, dn = stack.enter_context(skb.MultiFlow(devs)), None
        set_up(fl, dn, case)
        return fl, dn

    with contextlib.ExitStack() as stack:
        fl, dn = stepping(stack)
        if devs is not None:
            assert [fl.partition(g)[:2] for g in range(3)] == [(0, 1), (1, 2), (2, 3)]
        r0, (c0, q0) = fl.fibers(), fl.placement()
        bad = [dict(dt=0.0), dict(fiber_body=[0, 1, -1]), dict(site_ref=None), dict(num_blocks=301),
               dict(body_forces_torques=np.full((1, 6), np.inf))]
        for kw in bad:
            args = dict(dict(dt=0.02, fiber_body=case["fiber_body"], site_ref=case["site_ref"],
                             body_forces_torques=case["ft"], num_blocks=200), **kw)
            before = capi.launch_count()
            with pytest.raises(skb.SkbError, match="error 1:"):
                fl.step(*case_params(case), args.pop("dt"), ETA, dense=dn, **args)
            assert capi.launch_count() == before, kw
            c1, q1 = fl.placement()
            assert np.array_equal(fl.fibers(), r0) and np.array_equal(c0, c1) and np.array_equal(q0, q1), kw
        # and the links stay: a step after the refusals is the step from the untouched state
        x, tension, info = step_of(fl, dn, case)
        assert np.isfinite(info["fiber_error"])
        twin, dn2 = stepping(stack)
        x2, tension2, info2 = step_of(twin, dn2, case)
        assert np.array_equal(x, x2) and np.array_equal(tension, tension2) and info == info2
        assert np.array_equal(fl.fibers(), twin.fibers())
        assert all(np.array_equal(u, v) for u, v in zip(fl.placement(), twin.placement()))


def test_stepper_backs_up_and_restores_a_multiflow():
    case = step_case("FPB")
    with skb.MultiFlow([0, 0]) as mf:
        set_up(mf, None, case)
        s = timestep.Stepper(mf, None, case_params(case), ETA, fiber_body=case["fiber_body"],
                             site_ref=case["site_ref"], tol=1e-12, num_blocks=200, max_iters=400)
        r0, (c0, q0) = mf.fibers(), mf.placement()
        s.backup()
        i1 = s.step(0.02, body_forces_torques=case["ft"])
        r1, (c1, q1) = mf.fibers(), mf.placement()
        assert not np.array_equal(r1, r0) and not np.array_equal(q1, q0)
        s.restore()
        assert np.array_equal(mf.fibers(), r0) and np.array_equal(mf.placement()[1], q0)
        i2 = s.step(0.02, body_forces_torques=case["ft"])
        assert i1 == i2 and np.array_equal(mf.fibers(), r1) and np.array_equal(mf.placement()[1], q1)

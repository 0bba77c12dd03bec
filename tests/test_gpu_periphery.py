"""GPU tests of the periphery's shape (include/skelly_b200_flow.h skb_flow_set_periphery_shape,
skb_flow_periphery_interaction, and the step that applies it) against tests/periphery_reference.py.

FORCE BOUND, per node, from the long-double restatement (u = 2^-53, e = exp(-(R - |x|)/l_0), d = |dr|):
  eps_s = 8 u (|x| + R) + [ellipsoid] 8 u (a + b + c) / sin(theta)   the surface point and R: the roundings of the
          scaled point, its norm and the products (8 u (|x| + R)), and the CUDA ulp limits of atan2, acos, sin and cos
          (2 ulp each) with acos's 1 / sin(theta) conditioning in the polar angle (the 1e-12 guard keeps theta > 0)
  eps_r = 4 u |x|                                                       |x| (three squares, two adds, the root)
  |f_dev - f_ref|_k <= 2 f_0 e [ 2 (eps_s + eps_r) / d + (eps_s + eps_r + 4 u (R + |x|)) / l_0 + 12 u ]
the first term the |x| / |dr| amplification of dr = x - surface near the surface, the second the exp argument's
absolute error (exp itself: 1 ulp), the last the roundings of f_0 dr / d e; the factor 2 is spare.  Nodes within a
relative 1e-9 of the surface are excluded (their inside / outside decision may flip) and the test asserts how few."""
import contextlib

import numpy as np
import pytest

import periphery_reference as pr
import skellysim_b200 as skb
from skellysim_b200 import capi, timestep
from test_gpu_step import EMPTY, ETA, case_params, periphery, set_up, step_case

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
LD = np.longdouble
MARGIN = 1e-9
SPHERE = dict(kind="sphere", a=5.0, b=0.0, c=0.0, f_0=20.0, l_0=0.8, binding_active=1, polar_angle_start=0.3,
              polar_angle_end=2.2, binding_threshold=0.75)
ELLIPSOID = dict(SPHERE, kind="ellipsoid", a=7.8, b=4.16, c=4.16)  # the benchmark's C3 ellipsoid
KIND = {"sphere": capi.PERIPHERY_SPHERE, "ellipsoid": capi.PERIPHERY_ELLIPSOID}


def set_shape(fl, shape, **kw):
    fl.set_periphery_shape(KIND[shape["kind"]], shape["a"], shape["b"], shape["c"], shape["f_0"], shape["l_0"],
                           shape["binding_active"], shape["polar_angle_start"], shape["polar_angle_end"],
                           shape["binding_threshold"], **kw)


def ragged_fibers(shape, seed, n_fibers=40):
    """fibers of 8 to 128 nodes whose nodes lie inside, near and outside the shape"""
    rng = np.random.default_rng(seed)
    scale = np.array([shape["a"], shape["b"] or shape["a"], shape["c"] or shape["a"]])
    pos = []
    for _ in range(n_fibers):
        n = int(rng.integers(8, 129))
        d = rng.normal(size=3)
        d /= np.linalg.norm(d)
        start = d * scale * rng.uniform(0.2, 1.1)
        t = rng.normal(size=3)
        t /= np.linalg.norm(t)
        pos.append(start + np.linspace(0.0, rng.uniform(0.5, 3.0), n)[:, None] * t)
    return pos


@contextlib.contextmanager
def query_flow(pos, centers=EMPTY):
    """a flow with the fibers pos, a 60-node periphery and the bodies (one node each) at centers"""
    with skb.Flow(0) as fl:
        fl.set_fibers(np.concatenate(pos), [len(p) for p in pos], [1.0] * len(pos))
        r, nrm, _, _ = periphery(60, 5)
        fl.set_periphery(r, nrm)
        fl.set_bodies(np.asarray(centers, dtype=float).reshape(-1, 3), np.zeros((len(centers), 3)), centers)
        yield fl


def near_surface(shape, x, t=0.0):
    """nodes within a relative MARGIN of the surface shrunk by t"""
    x = np.asarray(x, dtype=LD)
    r = np.sqrt(np.sum(x * x, axis=1))
    if shape["kind"] == "sphere":
        R = np.full(len(x), LD(shape["a"]) - LD(t))
    else:
        rc = pr._cortex(shape, x, t, LD)
        R = np.sqrt(np.sum(rc * rc, axis=1))
    return np.abs(r - R) <= MARGIN * np.maximum(np.abs(R), 1)


def force_bound(shape, x):
    x = np.asarray(x, dtype=LD)
    r = np.sqrt(np.sum(x * x, axis=1))
    if shape["kind"] == "sphere":
        surf = x / r[:, None] * LD(shape["a"])
        R = np.full(len(x), LD(shape["a"]))
        eps_s = 8 * U * (r + R)
    else:
        surf = pr._cortex(shape, x, 0.0, LD)
        R = np.sqrt(np.sum(surf * surf, axis=1))
        rs = x / np.array([shape["a"], shape["b"], shape["c"]], dtype=LD)
        rs_mag = np.sqrt(np.sum(rs * rs, axis=1))
        sin_t = np.sin(np.arccos(rs[:, 2] / (LD(1e-12) + rs_mag)))
        eps_s = 8 * U * (r + R) + 8 * U * (shape["a"] + shape["b"] + shape["c"]) / sin_t
    d = np.sqrt(np.sum((x - surf) ** 2, axis=1))
    e = np.exp(-(R - r) / LD(shape["l_0"]))
    eps_r = 4 * U * r
    b = 2 * shape["f_0"] * e * (2 * (eps_s + eps_r) / d + (eps_s + eps_r + 4 * U * (R + r)) / shape["l_0"] + 12 * U)
    return np.asarray(b, dtype=np.float64)


@pytest.mark.parametrize("shape", [SPHERE, ELLIPSOID], ids=["sphere", "ellipsoid"])
def test_force_of_every_node_within_its_bound_and_the_flags_exact(shape):
    pos = ragged_fibers(shape, 7)
    clamped = (np.arange(len(pos)) % 3 == 0).astype(np.int32)  # every third fiber minus_clamped_
    with query_flow(pos) as fl:
        set_shape(fl, shape, fiber_minus_clamped=clamped)
        f, hinged, collided = fl.periphery_interaction()
    off = np.concatenate([[0], np.cumsum([len(p) for p in pos])])
    excluded = checked = 0
    for i, x in enumerate(pos):
        got = f[off[i]:off[i + 1]]
        want = np.asarray(pr.fiber_interaction(shape, x, bool(clamped[i]), LD))
        keep = ~near_surface(shape, x)
        excluded += int((~keep).sum())
        err = np.abs(got - want.astype(np.float64)).max(axis=1)
        bound = np.where(np.all(want == 0, axis=1), 0.0, force_bound(shape, x))
        assert np.all(err[keep] <= bound[keep]), (i, np.max(err[keep] - bound[keep]))
        checked += int(keep.sum())
        if not (near_surface(shape, x, shape["binding_threshold"]).any()
                or np.any(np.abs(pr.polar_angle(x[-1], LD) - np.array([shape["polar_angle_start"],
                                                                         shape["polar_angle_end"]])) <= MARGIN)):
            assert hinged[i] == pr.plus_hinged(shape, x, LD), i
        if clamped[i]:
            assert not got[0].any()
    assert checked > 2000 and excluded <= 2, (checked, excluded)
    assert 0 < hinged.sum() < len(pos)  # both decisions occur
    assert np.any(f != 0) and np.any(np.all(f == 0, axis=1))
    assert collided == pr.check_collision(shape, pos, [False] * len(pos), dtype=LD)
    assert collided  # some nodes lie outside


@pytest.mark.parametrize("shape", [SPHERE, ELLIPSOID], ids=["sphere", "ellipsoid"])
def test_collided_inside_and_outside(shape):
    inside = [np.linspace([0.0, 0.0, 0.0], [1.0, 1.0, 1.0], 16), np.linspace([-1.0, 0.5, 0.0], [-2.0, 1.0, 0.5], 8)]
    out = [inside[0], np.concatenate([inside[1], [[0.0, 0.0, 9.0]]])]
    for pos, want in ((inside, False), (out, True)):
        with query_flow(pos) as fl:
            set_shape(fl, shape)
            assert fl.periphery_interaction()[2] == want
    # node 0 beyond the surface: skipped for a minus-clamped fiber (before any step: fiber_minus_clamped)
    pos = [np.concatenate([[[0.0, 0.0, 9.0]], np.linspace([0.0, 0.0, 3.0], [0.0, 0.0, 1.0], 7)])]
    for clamp in (0, 1):
        with query_flow(pos) as fl:
            set_shape(fl, shape, fiber_minus_clamped=[clamp])
            assert fl.periphery_interaction()[2] == (not clamp)


def test_spherical_bodies_touching_and_separated():
    pos = [np.linspace([0.0, 0.0, 0.0], [0.5, 0.0, 0.0], 8)]
    c = np.array([[1.0, 0.0, 0.0], [3.0, 0.0, 0.0]])
    # separated, overlapping, one not spherical, |c| + r = 3.5 > R = 3.2, the same against the ellipsoid (its stub)
    cases = [([1.0, 0.9], False, SPHERE), ([1.0, 1.1], True, SPHERE), ([1.0, 0.0], False, SPHERE),
             ([2.5, 0.0], True, dict(SPHERE, a=3.2)), ([2.5, 0.0], False, ELLIPSOID)]
    for radius, want, shp in cases:
        with query_flow(pos, c) as fl:
            set_shape(fl, shp, body_radius=radius)
            assert fl.periphery_interaction()[2] == want, (radius, shp["kind"])
            assert want == pr.bodies_collided(shp, c, radius)


# ---- the step ----------------------------------------------------------------------------------------------------------
STEP_SHAPE = dict(SPHERE, a=12.0, f_0=2.0, l_0=3.0, polar_angle_start=0.0, polar_angle_end=np.pi / 2,
                  binding_threshold=9.0)


def shaped_case():
    case = step_case("FPB")
    n_fib = sum(len(p) for p in case["fibers"])
    case["f_ext"] = 0.1 * np.random.default_rng(4).normal(size=(n_fib, 3))
    return case


def step(fl, dn, case, f_ext, plus_hinged=0, dt=0.02):
    p = case_params(case)[:-1] + (plus_hinged,)
    return fl.step(*p, dt, ETA, dense=dn, f_external=f_ext, body_forces_torques=case["ft"],
                   fiber_body=case["fiber_body"], site_ref=case["site_ref"], tol=1e-12, num_blocks=200, max_iters=400)


def without(info, key="collided"):
    return {k: v for k, v in info.items() if k != key}


def test_the_step_with_a_shape_is_the_step_with_its_force_and_binding():
    """bitwise: x, tension, info and the new geometry over three steps, against a twin that is handed the caller's
    f_external + periphery_interaction()'s force and its plus_hinged"""
    case = shaped_case()
    with contextlib.ExitStack() as stack:
        fl, twin = stack.enter_context(skb.Flow(0)), stack.enter_context(skb.Flow(0))
        dn, dn2 = stack.enter_context(skb.Dense(device_ids=[0])), stack.enter_context(skb.Dense(device_ids=[0]))
        set_up(fl, dn, case)
        set_up(twin, dn2, case)
        set_shape(fl, STEP_SHAPE, body_radius=[0.5])
        seen_hinged = 0
        for k in range(3):
            f, hinged, _ = fl.periphery_interaction()
            seen_hinged += int(hinged.sum())
            x, t, info = step(fl, dn, case, case["f_ext"])
            x2, t2, info2 = step(twin, dn2, case, case["f_ext"] + f, plus_hinged=hinged)
            assert np.array_equal(x, x2) and np.array_equal(t, t2), k
            assert without(info) == without(info2) and info["collided"] == 0 and info2["collided"] == 0, k
            assert np.array_equal(fl.fibers(), twin.fibers())
            assert all(np.array_equal(a, b) for a, b in zip(fl.placement(), twin.placement()))
            assert np.abs(f).max() > 1e-3  # the repulsion is not negligible
        assert seen_hinged > 0
        # NULL f_external: the repulsion alone
        f, hinged, _ = fl.periphery_interaction()
        x, t, info = step(fl, dn, case, None)
        x2, t2, info2 = step(twin, dn2, case, f, plus_hinged=hinged)
        assert np.array_equal(x, x2) and np.array_equal(t, t2) and without(info) == without(info2)


def crossing_radius(case, pick):
    """a sphere radius that the step of `case` (without a shape) crosses: between pick(before) and pick(after)"""
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0]))
        set_up(fl, dn, case)
        before = pick(fl)
        step(fl, dn, case, case["f_ext"])
        after = pick(fl)
    assert after > before + 1e-4, (before, after)
    return before, after


def test_collided_after_a_step_that_crosses_the_surface_and_run_halves_dt():
    case = shaped_case()
    fiber_r = lambda fl: np.linalg.norm(fl.fibers(), axis=1).max()
    body_c = lambda fl: np.linalg.norm(fl.placement()[0][0])
    # (tiny f_0: the repulsion moves nothing by the margins below)
    weak = dict(STEP_SHAPE, f_0=1e-12, binding_active=0)
    b0, b1 = crossing_radius(case, fiber_r)
    c0, c1 = crossing_radius(case, body_c)
    R_fib = 0.5 * (b0 + b1)
    for shape, radius, want in ((dict(weak, a=R_fib), [0.0], 1), (dict(weak, a=20.0), [20.0 - 0.5 * (c0 + c1)], 1),
                                (dict(weak, a=20.0), [0.5], 0)):
        with contextlib.ExitStack() as stack:
            fl = stack.enter_context(skb.Flow(0))
            dn = stack.enter_context(skb.Dense(device_ids=[0]))
            set_up(fl, dn, case)
            set_shape(fl, shape, body_radius=radius)
            assert not fl.periphery_interaction()[2]
            _, _, info = step(fl, dn, case, case["f_ext"])
            assert info["converged"] and info["collided"] == want, (shape["a"], radius)
    # timestep.run rejects the colliding step, restores and halves dt
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0]))
        set_up(fl, dn, case)
        set_shape(fl, dict(weak, a=b0 + 0.75 * (b1 - b0)))  # dt 0.02 crosses it, dt 0.01 does not
        r0 = fl.fibers()
        s = timestep.Stepper(fl, dn, case_params(case), ETA, fiber_body=case["fiber_body"], site_ref=case["site_ref"],
                             tol=1e-12, num_blocks=200, max_iters=400)
        forces = lambda time, r: (case["f_ext"], case["ft"])
        _, dt, log = timestep.run(s, 0.01, 0.02, dt_min=1e-4, fiber_error_tol=10.0, forces=forces)
        assert [(d, acc) for _, d, acc, _ in log] == [(0.02, False), (0.01, True)], log
        assert not np.array_equal(r0, fl.fibers())
        # a caller's callable takes precedence
        s2 = timestep.Stepper(fl, dn, case_params(case), ETA, fiber_body=case["fiber_body"],
                              site_ref=case["site_ref"], tol=1e-12, num_blocks=200, max_iters=400)
        _, _, log2 = timestep.run(s2, 0.01, 0.005, fiber_error_tol=10.0, forces=forces,
                                  collided=lambda r, c: False)
        assert all(acc for _, _, acc, _ in log2)


def test_mflow_and_the_group_step_apply_the_shape():
    """[0]: bitwise the single-device step with the shape; [0, 0]: bitwise the [0, 0] step handed the force and the
    binding; the group step (RankStepper) bitwise skb_mflow_step with the shape, the same collided on every member, and
    no allocation inside the step.  [0, 0] is held to a [0, 0] twin, not to the single device: without a shape too,
    two members reduce the solve's dot products in another order than one device, so their steps agree with the
    single device's within the solve's tolerance only (test_gpu_step.test_mflow_steps_as_the_single_device)"""
    from test_gpu_group_step import Ranks, check_members, mflow_step
    case = shaped_case()
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0]))
        set_up(fl, dn, case)
        set_shape(fl, STEP_SHAPE, body_radius=[0.5])
        single = [step(fl, dn, case, case["f_ext"]) for _ in range(2)]
    with skb.MultiFlow([0]) as mf:
        set_up(mf, None, case)
        set_shape(mf, STEP_SHAPE, body_radius=[0.5])
        for k in range(2):
            x, t, info = step(mf, None, case, case["f_ext"])
            assert np.array_equal(x, single[k][0]) and np.array_equal(t, single[k][1]) and info == single[k][2]
    with skb.MultiFlow([0, 0]) as mf, skb.MultiFlow([0, 0]) as twin:
        set_up(mf, None, case)
        set_up(twin, None, case)
        set_shape(mf, STEP_SHAPE, body_radius=[0.5])
        for k in range(2):
            f, hinged, _ = mf.periphery_interaction()
            x, t, info = step(mf, None, case, case["f_ext"])
            x2, t2, info2 = step(twin, None, case, case["f_ext"] + f, plus_hinged=hinged)
            assert np.array_equal(x, x2) and np.array_equal(t, t2) and without(info) == without(info2), k
            assert np.array_equal(mf.fibers(), twin.fibers())
    with skb.MultiFlow([0, 0]) as mf:
        R = Ranks([0, 0], case)
        try:
            set_up(mf, None, case)
            set_shape(mf, STEP_SHAPE, body_radius=[0.5])
            for g in R.flows:
                set_shape(g, STEP_SHAPE, body_radius=[0.5])
            for k in range(2):
                infos = R.step()  # (asserts that no device memory was allocated)
                x, tension, info = mflow_step(mf, case)
                check_members(R, infos, x, tension, info, mf)
                assert len({i["collided"] for i in infos}) == 1
        finally:
            R.close()


def test_refusals_keep_the_earlier_shape():
    pos = [np.linspace([0.5, 0.0, 0.0], [1.5, 0.0, 0.0], 8), np.linspace([0.0, 0.0, 4.5], [0.0, 0.0, 5.5], 8)]
    with query_flow(pos, np.zeros((1, 3))) as fl:
        set_shape(fl, SPHERE)
        ref = fl.periphery_interaction()
        bad = [dict(kind=3), dict(a=np.nan), dict(f_0=np.inf), dict(a=0.0), dict(l_0=0.0), dict(l_0=-1.0),
               dict(binding_active=2)]
        for kw in bad:
            args = dict(kind=KIND["sphere"], a=5.0, b=0.0, c=0.0, f_0=20.0, l_0=0.8, binding_active=1,
                        polar_angle_start=0.3, polar_angle_end=2.2, binding_threshold=0.75)
            args.update(kw)
            with pytest.raises(skb.SkbError):
                fl.set_periphery_shape(**args)
        for kw in (dict(kind=KIND["ellipsoid"], a=7.8, b=0.0, c=4.16), dict(kind=KIND["ellipsoid"], a=7.8, b=4.16,
                                                                            c=-1.0)):
            with pytest.raises(skb.SkbError):
                fl.set_periphery_shape(**kw)
        with pytest.raises(skb.SkbError):
            set_shape(fl, SPHERE, fiber_minus_clamped=[0, 2])
        for r in ([-1.0], [np.nan], [np.inf]):
            with pytest.raises(skb.SkbError):
                set_shape(fl, SPHERE, body_radius=r)
        got = fl.periphery_interaction()
        assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]) and got[2] == ref[2]
        fl.set_periphery_shape(capi.PERIPHERY_NONE, 0.0)
        with pytest.raises(skb.SkbError, match="no periphery shape"):
            fl.periphery_interaction()
    with skb.Flow(0) as fl:  # no periphery nodes
        fl.set_fibers(pos[0], [8], [1.0])
        fl.set_periphery(EMPTY, EMPTY)
        fl.set_bodies(EMPTY, EMPTY, EMPTY)
        with pytest.raises(skb.SkbError, match="no periphery nodes"):
            set_shape(fl, SPHERE)


def test_a_step_refuses_a_shape_its_fibers_outgrew_and_a_non_finite_force():
    case = shaped_case()
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0]))
        set_up(fl, dn, case)
        set_shape(fl, STEP_SHAPE, body_radius=[0.5])
        more = dict(case, fibers=case["fibers"] + [case["fibers"][2] + 0.5], lengths=case["lengths"] + [0.8],
                    fiber_body=case["fiber_body"] + [-1], site_ref=np.concatenate([case["site_ref"], np.zeros((1, 3))]),
                    clamped=case["clamped"] + [0])
        more["f_ext"] = np.zeros((sum(len(p) for p in more["fibers"]), 3))
        fl.set_fibers(np.concatenate(more["fibers"]), [16] * 4, more["lengths"])
        fl.set_gmres(300)
        r0 = fl.fibers()
        with pytest.raises(skb.SkbError, match="skb_flow_set_periphery_shape"):
            step(fl, dn, more, more["f_ext"])
        assert np.array_equal(fl.fibers(), r0)
        set_shape(fl, STEP_SHAPE, body_radius=[0.5])
        _, _, info = step(fl, dn, more, more["f_ext"])
        assert info["converged"]
    # a node at the centre of a sphere: 0 / 0 in the reference, refused by the step with the geometry untouched
    case = step_case("FP")
    case["fibers"][0] = case["fibers"][0] - case["fibers"][0][3]
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0]))
        set_up(fl, dn, case)
        set_shape(fl, STEP_SHAPE)
        f, _, _ = fl.periphery_interaction()
        assert np.isnan(f[3]).all() and np.isfinite(np.delete(f, 3, axis=0)).all()
        r0 = fl.fibers()
        with pytest.raises(skb.SkbError, match="non-finite fiber-periphery force"):
            step(fl, dn, case, None)
        assert np.array_equal(fl.fibers(), r0)


def bound_outside_case():
    """a body at (2, 0, 0) with one fiber bound at (1.5, 0, 0) pointing to the origin, and one free fiber near the
    origin: node 0 of the bound fiber lies beyond the ellipsoid OUTSIDE_SHAPE, every other node inside it"""
    rng = np.random.default_rng(31)
    from test_gpu_step import random_unit_quaternion
    import step_reference as st
    q0 = random_unit_quaternion(rng)
    c0 = np.array([2.0, 0.0, 0.0])
    Rq = st.rotation(q0)
    site_ref = np.array([Rq.T @ np.array([-0.5, 0.0, 0.0]), np.zeros(3)])
    t = np.linspace(0.0, 0.8, 16)[:, None]
    pos = [c0 + Rq @ site_ref[0] + t * np.array([-1.0, 0.0, 0.0]),
           np.array([-1.0, 0.5, 0.0]) + t * np.array([0.0, 0.6, 0.8])]
    case = dict(fibers=pos, lengths=[0.8, 0.8], body=dict(n=100, R=0.5, c0=c0, q0=q0), n_shell=60,
                fiber_body=[0, -1], site_ref=site_ref, clamped=[1, 0], ft=None)
    case["f_ext"] = np.zeros((32, 3))
    return case


OUTSIDE_SHAPE = dict(ELLIPSOID, a=1.475, f_0=1e-6, binding_active=0)


def test_every_group_member_skips_node_0_of_the_same_clamped_fibers():
    """the bound fiber is clamped (params minus_clamped) but not minus_clamped_ (fiber_minus_clamped 0), and its node 0
    lies beyond the ellipsoid (whose body test is the reference's stub).  A member that does not own it learns its
    clamp through the step's all-gather: every member reports collided = 0, as skb_mflow_step does; and the first
    member owns the bound fiber, the second the free one"""
    from test_gpu_group_step import Ranks, check_members, mflow_step
    case = bound_outside_case()
    with skb.MultiFlow([0, 0]) as mf:
        R = Ranks([0, 0], case)
        try:
            assert [p[:2] for p in R.parts] == [(0, 1), (1, 2)], R.parts
            set_up(mf, None, case)
            for fl in [mf] + R.flows:
                set_shape(fl, OUTSIDE_SHAPE, body_radius=[0.5])
            assert mf.periphery_interaction()[2]  # before a step only fiber_minus_clamped is known: node 0 counts
            for k in range(2):
                infos = R.step()
                x, tension, info = mflow_step(mf, case)
                check_members(R, infos, x, tension, info, mf)
                assert [i["collided"] for i in infos] == [0, 0] and info["collided"] == 0, k
                r = mf.fibers()
                assert pr.outside(OUTSIDE_SHAPE, r[:1]).all() and not pr.outside(OUTSIDE_SHAPE, r[1:]).any(), k
            assert not mf.periphery_interaction()[2]
        finally:
            R.close()


def test_a_refused_step_leaves_the_collision_test_as_it_was():
    """node 0 beyond the sphere, the fiber minus_clamped_ = 0 but clamped in the step's params: a refused step (a
    non-finite f_external) records nothing; an installed one records the clamp, and node 0 no longer counts"""
    pos = [np.linspace([0.0, 0.0, 3.5], [0.0, 0.0, 1.0], 16)]
    case = dict(fibers=pos, lengths=[2.5], body=None, n_shell=60, fiber_body=None, site_ref=None, clamped=[1], ft=None)
    shape = dict(SPHERE, a=3.4, f_0=1e-6, binding_active=0)
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0]))
        set_up(fl, dn, case)
        set_shape(fl, shape, fiber_minus_clamped=[0])
        assert fl.periphery_interaction()[2]
        bad = np.zeros((16, 3))
        bad[5, 1] = np.nan
        with pytest.raises(skb.SkbError, match="non-finite external force"):
            step(fl, dn, case, bad)
        assert fl.periphery_interaction()[2]
        _, _, info = step(fl, dn, case, np.zeros((16, 3)))
        r = fl.fibers()
        assert pr.outside(shape, r[:1]).all() and not pr.outside(shape, r[1:]).any()
        assert info["collided"] == 0 and not fl.periphery_interaction()[2]

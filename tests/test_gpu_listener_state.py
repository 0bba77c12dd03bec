"""GPU tests of skb_flow_set_listener_state(_device) (include/skelly_b200_flow.h): the listener's frame built on the
device from the installed geometry and a step's solution.  Bitwise against the public calls a caller composes today
(the same kernels); against tests/listener_state_reference.py through the oracle's flows at the 1e-12 gate; after a
real skb_flow_step; on empty blocks; every refusal leaving no frame; and timestep.run's observe callback.

Fibers are kept to n <= 32 nodes, lengths in [1, 2] and positions within a box of 2 and tensions of order 10: there
the fiber forces' own rounding (the fourth-derivative rows of force_operator_ cancel on a nearly straight fiber) stays
below 1e-13 of their scale, so that the gate tests the frame and not the conditioning of apply_fiber_force."""
import contextlib

import numpy as np
import pytest

import listener_state_reference as lsr
import skellysim_b200 as skb
import step_reference as st
import streamline_reference as sl
from conftest import rel_max
from skellysim_b200 import capi, timestep
from test_gpu_listener import Frame, clear_seeds
from test_gpu_step import case_params, fiber_flow, set_classes, set_up, step_case, step_of, straight_fibers
from test_gpu_system_edges import sphere

pytestmark = pytest.mark.gpu
ETA, DT = 0.9, 1e-3
EMPTY = np.zeros((0, 3))
SHAPE = dict(kind="sphere", a=4.5, b=0.0, c=0.0, f_0=2.0, l_0=0.5, binding_active=0, polar_angle_start=0.0,
             polar_angle_end=np.pi, binding_threshold=0.75)


def make(seed, n_fibers, n_shell, n_body_nodes, n_bodies, bound=True, nodes=(16, 24, 32)):
    """fibers (every third bound, when bound and there are bodies), a periphery of n_shell nodes, n_bodies bodies of
    n_body_nodes / n_bodies nodes, point sources and a background; a random solution and tension"""
    rng = np.random.default_rng(seed)
    n_nodes = [int(n) for n in rng.choice(nodes, size=n_fibers)] if n_fibers else []
    pos, lengths = [], []
    for n in n_nodes:
        L = rng.uniform(1.0, 2.0)
        t = rng.normal(size=3)
        t /= np.linalg.norm(t)
        s = np.linspace(0.0, L, n)
        bend = np.cross(t, rng.normal(size=3))
        pos.append(rng.uniform(-2, 2, 3) + s[:, None] * t + 0.05 * np.sin(3 * s)[:, None] * bend)
        lengths.append(L)
    d = rng.normal(size=(n_shell, 3))
    d /= np.linalg.norm(d, axis=1)[:, None] if n_shell else 1
    per = n_body_nodes // max(n_bodies, 1)
    centers = rng.uniform(-2, 2, (n_bodies, 3))
    e = [rng.normal(size=(per, 3)) for _ in range(n_bodies)]
    e = [v / np.linalg.norm(v, axis=1)[:, None] for v in e]
    sd = dict(
        fib=dict(pos=np.concatenate(pos) if pos else EMPTY, n_nodes=n_nodes, lengths=np.array(lengths)),
        shell=dict(pos=d * np.array([7.8, 4.16, 4.16]), normals=-d),
        body=dict(pos=np.concatenate([c + 0.4 * v for c, v in zip(centers, e)]) if n_bodies else EMPTY,
                  normals=np.concatenate(e) if n_bodies else EMPTY, centers=centers, n_nodes=[per] * n_bodies),
        kind=np.array([1, 2] * n_bodies, dtype=np.int32)[:n_bodies], radii=np.tile([0.4, 0.5, 0.3], (n_bodies, 1)),
        pts=rng.uniform(-1, 1, (2, 3)), bg=([1, 0, 2], np.array([0.2, -0.1, 0.05]), np.array([0.05, 0.0, -0.02])))
    sd["pf"], sd["ptq"] = 0.3 * rng.normal(size=(2, 3)), 0.3 * rng.normal(size=(2, 3))
    body = np.array([(f // 3) % n_bodies if (bound and n_bodies and f % 3 == 0) else -1 for f in range(n_fibers)])
    sd["links"] = dict(body=body, site=np.array([p[0] for p in pos]) if pos else EMPTY,
                       rigidity=np.full(n_fibers, 2.5e-3))
    sd["params"] = (sd["fib"]["lengths"], 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)
    n_x = 4 * sum(n_nodes) + 3 * n_shell + n_bodies * (3 * per + 6)
    sd["x"], sd["tension"] = rng.uniform(-1, 1, n_x), rng.uniform(-10, 10, sum(n_nodes))
    sd["w"] = rng.uniform(0.5, 1.0, n_bodies * per)
    sd["ex"], sd["ey"], sd["ez"] = (rng.uniform(-1, 1, (n_bodies * per, 3)) for _ in range(3))
    return sd


@contextlib.contextmanager
def opened(sd, shape=True, links=True, derivatives=True):
    with skb.Flow(0) as fl:
        fib, shell, body = sd["fib"], sd["shell"], sd["body"]
        fl.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
        fl.set_periphery(shell["pos"], shell["normals"])
        fl.set_bodies(body["pos"], body["normals"], body["centers"])
        if derivatives:
            set_classes(fl, fib["n_nodes"])
        else:
            from oracle.fiber_fd import compute_matrices
            for n in sorted(set(fib["n_nodes"])):
                m = compute_matrices(n)
                fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_body_operators(body["n_nodes"], sd["w"], sd["ex"], sd["ey"], sd["ez"])
        if links and fl.n_bodies and len(fib["n_nodes"]):
            fl.set_fiber_links(sd["links"]["body"], sd["links"]["site"], sd["links"]["rigidity"])
        if shape and len(shell["pos"]):
            fl.set_periphery_shape(capi.PERIPHERY_SPHERE, SHAPE["a"], f_0=SHAPE["f_0"], l_0=SHAPE["l_0"])
        fl.set_point_sources(sd["pts"], sd["pf"], sd["ptq"])
        fl.set_background(*sd["bg"])
        yield fl


def set_state(fl, sd, flag):
    capi.set_listener_state(fl, *sd["params"], DT, ETA, sd["tension"], sd["x"], sd["kind"], sd["radii"], flag)


def restated(sd, flag):
    """the restatement's frame as a test_gpu_listener.Frame, whose velocity() is the oracle's"""
    out = lsr.frame(sd["fib"], len(sd["shell"]["pos"]), sd["body"], sd["links"], sd["params"], DT, ETA, sd["x"],
                    sd["tension"], shape=SHAPE, periphery_interaction=flag)
    fr = Frame.__new__(Frame)
    fr.fib = dict(sd["fib"], forces=out["fib_forces"])
    fr.shell = dict(sd["shell"], density=out["shell_density"])
    fr.body = dict(sd["body"], density=out["body_densities"], forces=out["body_ft"][:, :3],
                   torques=out["body_ft"][:, 3:])
    fr.kind, fr.radii, fr.uw = sd["kind"], sd["radii"], out["body_uw"]
    fr.pts, fr.pf, fr.ptq, fr.bg = sd["pts"], sd["pf"], sd["ptq"], sd["bg"]
    return fr, out


def targets(sd, rng, n=600):
    c = sd["body"]["centers"]
    inside = [c[b] + rng.uniform(-0.15, 0.15, (20, 3)) for b in range(len(c))]
    return np.concatenate([rng.uniform(-3, 3, (n, 3))] + inside)


def check(v, fr, r):
    """the 1e-12 gate outside the bodies; inside each body exactly its rigid motion"""
    ref = fr.velocity(r)
    ins = fr.inside(r) if len(fr.body["centers"]) else []
    free = np.ones(len(r), dtype=bool)
    for m in ins:
        free &= ~m
    assert rel_max(v[free], ref[free]) <= 1e-12, rel_max(v[free], ref[free])
    for b, m in enumerate(ins):
        assert m.any() and np.array_equal(v[m], ref[m]), b


@pytest.mark.parametrize("bound", [False, True])
@pytest.mark.parametrize("flag", [False, True])
def test_the_frame_is_the_public_composition_bitwise(flag, bound):
    """The state call's frame against skb_flow_set_listener_frame fed what the public calls give: apply_fiber_force of
    the packed [x; T] after build_fiber_operators (+ the repulsion of periphery_interaction), the solution's slices, and
    zero body forces and torques.  Bound fibers take the link kernel's path with forces and torques exactly zero: zero
    link rigidity and zero tension at their node 0.  Targets beside every fiber node make each node's force show."""
    sd = make(3, 9, 180, 120, 2, bound=bound)
    off = np.concatenate([[0], np.cumsum(sd["fib"]["n_nodes"])])
    if bound:
        b = sd["links"]["body"] >= 0
        assert b.any()
        sd["links"]["rigidity"][:] = 0.0
        sd["tension"][off[:-1][b]] = 0.0
        assert np.array_equal(restated(sd, flag)[1]["body_ft"], np.zeros((2, 6)))
    rng = np.random.default_rng(1)
    r = np.concatenate([targets(sd, rng), sd["fib"]["pos"] + rng.uniform(-0.02, 0.02, sd["fib"]["pos"].shape)])
    with opened(sd) as fl:
        set_state(fl, sd, flag)
        v_state = fl.velocity_field(r)
        packed = np.concatenate([np.concatenate([sd["fib"]["pos"][a:b].T.reshape(-1), sd["tension"][a:b]])
                                 for a, b in zip(off[:-1], off[1:])])
        fl.build_fiber_operators(*sd["params"], DT, ETA)
        ff = fl.apply_fiber_force(packed)
        if flag:
            rep = fl.periphery_interaction()[0]
            assert np.abs(rep).max() > 0  # the repulsion is there
            ff = ff + rep
        nf, ns = 4 * int(off[-1]), len(sd["shell"]["pos"])
        xs, xb = sd["x"][nf:nf + 3 * ns], sd["x"][nf + 3 * ns:]
        per = sd["body"]["n_nodes"][0]
        blocks = xb.reshape(2, 3 * per + 6)
        fl.set_listener_frame(ff, xs.reshape(-1, 3), blocks[:, :3 * per].reshape(-1, 3), np.zeros((2, 6)),
                              blocks[:, 3 * per:], sd["kind"], sd["radii"], ETA)
        v_frame = fl.velocity_field(r)
    assert np.array_equal(v_state, v_frame)


def test_the_host_and_device_forms_are_bitwise_equal():
    torch = pytest.importorskip("torch")
    sd = make(4, 12, 150, 100, 2)
    r = targets(sd, np.random.default_rng(2))
    with opened(sd) as fl:
        set_state(fl, sd, True)
        v_host = fl.velocity_field(r)
        dx = torch.from_numpy(sd["x"]).cuda()
        dt_ = torch.from_numpy(sd["tension"]).cuda()
        stream = torch.cuda.current_stream().cuda_stream
        capi.set_listener_state_device(fl, *sd["params"], DT, ETA, dt_.data_ptr(), dx.data_ptr(), sd["kind"],
                                       sd["radii"], True, stream=stream)
        v_dev = fl.velocity_field(r)
    assert np.array_equal(v_host, v_dev)


def test_the_state_leaves_the_operators_without_their_inverse():
    """the frame's build assembles A_, force_operator_ and xs_ only: the fiber preconditioner refuses until a build with
    the inverse, and the operators it left are those of skb_flow_build_fiber_operators"""
    sd = make(10, 6, 0, 0, 0)
    with opened(sd) as fl:
        set_state(fl, sd, False)
        x = np.random.default_rng(3).uniform(-1, 1, 4 * fl.n_fib)
        with pytest.raises(skb.SkbError, match="error 1:.*preconditioner"):
            fl.apply_fiber_preconditioner(x)
        ops = fl.get_fiber_operators(inverse=False)
        fl.build_fiber_operators(*sd["params"], DT, ETA)
        full = fl.get_fiber_operators(inverse=False)
        fl.apply_fiber_preconditioner(x)
    for k in ("A", "force"):
        assert all(np.array_equal(a, b) for a, b in zip(ops[k], full[k]))
    assert np.array_equal(ops["xs"], full["xs"])


def test_the_velocity_field_matches_the_restatement():
    # free and bound fibers, a sphere and an ellipsoid interior, a periphery with a shape, point sources, a background.
    # One size: the listener's evaluations take the plain pair kernel whatever the size (velocity_dev never takes the
    # matvec's symmetric or cross path), so a larger system runs no other code
    sd = make(5, 12, 200, 160, 2)
    fr, out = restated(sd, True)
    assert np.abs(out["body_ft"]).max() > 0 and (sd["links"]["body"] < 0).any()
    r = targets(sd, np.random.default_rng(3))
    with opened(sd) as fl:
        set_state(fl, sd, True)
        v = fl.velocity_field(r)
    check(v, fr, r)


def test_after_a_real_step_the_frame_is_the_installed_state():
    case = step_case("FPB")
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0]))
        set_up(fl, dn, case)
        x, tension, info = step_of(fl, dn, case)
        assert info["converged"]
        kind, radii = np.array([1], dtype=np.int32), np.array([[0.5, 0.5, 0.5]])
        capi.set_listener_state(fl, *case_params(case), 0.02, ETA, tension, x, kind, radii)
        # the restatement at the installed geometry: the fibers, the placed body and its sites
        c, q = fl.placement()
        R = st.rotation(q[0])
        r_ref, n_ref, _ = sphere(case["body"]["n"], case["body"]["R"])
        from test_gpu_step import periphery
        r_sh, n_sh, _, _ = periphery(case["n_shell"], 5)
        nodes = [len(p) for p in case["fibers"]]
        sd = dict(fib=dict(pos=fl.fibers(), n_nodes=nodes, lengths=np.asarray(case["lengths"])),
                  shell=dict(pos=r_sh, normals=n_sh),
                  body=dict(pos=c[0] + r_ref @ R.T, normals=n_ref @ R.T, centers=c, n_nodes=[case["body"]["n"]]),
                  links=dict(body=np.array(case["fiber_body"]),
                             site=np.array([st.site(c[0], q[0], s) for s in case["site_ref"]]),
                             rigidity=np.full(3, 2.5e-3)),
                  params=case_params(case), x=x, tension=tension, kind=kind, radii=radii,
                  pts=np.zeros((0, 3)), pf=np.zeros((0, 3)), ptq=np.zeros((0, 3)),
                  bg=([0, 1, 2], np.zeros(3), np.array([0.3, -0.2, 0.5])))
        out = lsr.frame(sd["fib"], case["n_shell"], sd["body"], sd["links"], sd["params"], 0.02, ETA, x, tension)
        fr = Frame.__new__(Frame)
        fr.fib = dict(sd["fib"], forces=out["fib_forces"])
        fr.shell = dict(sd["shell"], density=out["shell_density"])
        fr.body = dict(sd["body"], density=out["body_densities"], forces=out["body_ft"][:, :3],
                       torques=out["body_ft"][:, 3:])
        fr.kind, fr.radii, fr.uw = kind, radii, out["body_uw"]
        fr.pts, fr.pf, fr.ptq, fr.bg = sd["pts"], sd["pf"], sd["ptq"], sd["bg"]
        rng = np.random.default_rng(4)
        r = np.concatenate([rng.uniform(-2, 2, (300, 3)), c[0] + rng.uniform(-0.2, 0.2, (20, 3))])
        check(fl.velocity_field(r), fr, r)
        x0 = clear_seeds(fr, np.random.default_rng(5), 3)
        got = fl.streamlines(x0, t_final=0.5)
        ref = sl.lines(fr.velocity, x0, t_final=0.5, max_points=1000)
        for g, e in zip(got, ref):
            assert len(g["time"]) == len(e["time"]) and g["status"] == e["status"]
            assert np.abs(g["x"] - e["x"]).max() <= 1e-9 * max(1.0, np.abs(e["x"]).max())
        # a further step installs a new geometry: the frame is stale
        step_of(fl, dn, case)
        with pytest.raises(skb.SkbError, match="error 4:"):
            fl.velocity_field(r)
        with pytest.raises(skb.SkbError, match="error 4:"):
            fl.streamlines(x0)


@pytest.mark.parametrize("shape", [(12, 0, 0, 0), (0, 150, 0, 0), (0, 0, 80, 2), (0, 0, 0, 0)])
def test_empty_blocks_need_none_of_their_set_up(shape):
    sd = make(8, *shape)
    fr, _ = restated(sd, False)
    r = targets(sd, np.random.default_rng(6), 200)
    with skb.Flow(0) as fl:
        # only what the non-empty blocks need
        fib, shell, body = sd["fib"], sd["shell"], sd["body"]
        fl.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
        fl.set_periphery(shell["pos"], shell["normals"])
        fl.set_bodies(body["pos"], body["normals"], body["centers"])
        if fib["n_nodes"]:
            set_classes(fl, fib["n_nodes"])
        if body["n_nodes"]:
            fl.set_body_operators(body["n_nodes"], sd["w"], sd["ex"], sd["ey"], sd["ez"])
        fl.set_point_sources(sd["pts"], sd["pf"], sd["ptq"])
        fl.set_background(*sd["bg"])
        L = capi.library()
        p = capi.fiber_params(len(fib["n_nodes"]), *sd["params"])
        null = lambda a, n: capi._p(a) if n else None  # noqa: E731
        kind = sd["kind"].ctypes.data_as(capi.C.POINTER(capi.C.c_int32)) if len(sd["kind"]) else None
        rc = L.skb_flow_set_listener_state(fl._h, capi._params_ptr(p), DT, ETA, null(sd["tension"], fib["n_nodes"]),
                                           null(sd["x"], len(sd["x"])), kind, null(sd["radii"], len(sd["kind"])), 0)
        assert rc == 0, L.skb_last_error_string()
        v = fl.velocity_field(r)
    check(v, fr, r)


def _refused(fl, sd, code=1, **kw):
    args = dict(params=sd["params"], dt=DT, eta=ETA, tension=sd["tension"], x=sd["x"], kind=sd["kind"],
                radii=sd["radii"], flag=True)
    args.update(kw)
    set_state(fl, sd, True)
    fl.velocity_field(np.zeros((1, 3)))
    with pytest.raises(skb.SkbError, match=f"error {code}:"):
        capi.set_listener_state(fl, *args["params"], args["dt"], args["eta"], args["tension"], args["x"], args["kind"],
                              args["radii"], args["flag"])
    with pytest.raises(skb.SkbError, match="error 4:"):  # no frame is left
        fl.velocity_field(np.zeros((1, 3)))


def test_each_refusal_leaves_no_frame():
    sd = make(9, 6, 100, 80, 2)
    bad_t = sd["tension"].copy()
    bad_t[3] = np.nan
    with opened(sd) as fl:
        _refused(fl, sd, dt=np.nan)
        _refused(fl, sd, dt=0.0)
        _refused(fl, sd, eta=0.0)
        _refused(fl, sd, eta=np.inf)
        _refused(fl, sd, tension=bad_t)
        _refused(fl, sd, kind=np.array([3, 1], dtype=np.int32))
        _refused(fl, sd, radii=np.zeros((2, 3)))
        _refused(fl, sd, params=(sd["params"][0], 2.5e-3, 0.0, 500.0, 1.0, 0, 0))  # radius 0
    with opened(sd, links=False) as fl:
        with pytest.raises(skb.SkbError, match="error 1:.*set_fiber_links"):
            set_state(fl, sd, True)
    with opened(sd, shape=False) as fl:
        with pytest.raises(skb.SkbError, match="error 1:.*periphery_shape"):
            set_state(fl, sd, True)
        set_state(fl, sd, False)  # (no shape is needed without the flag)
    with opened(sd, links=False, derivatives=False) as fl:
        with pytest.raises(skb.SkbError, match="error 1:.*derivatives"):
            set_state(fl, sd, True)
    with opened(sd) as fl:
        # the links are dropped with the geometry: set for the current geometry only
        fl.set_fibers(sd["fib"]["pos"], sd["fib"]["n_nodes"], sd["fib"]["lengths"])
        with pytest.raises(skb.SkbError, match="error 1:.*set_fiber_links"):
            set_state(fl, sd, True)


def test_run_observes_every_accepted_step_and_changes_no_step():
    pos, lengths = straight_fibers(3, 16, 71)
    p = (np.asarray(lengths), 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)
    seen = []

    def observe(time, stepper, info):
        stepper.set_listener_state()
        seen.append((time, stepper.flow.velocity_field(np.array([[1.5, 5.0, -4.0]]))[0].copy(), info["fiber_error"]))

    results = []
    for obs in (None, observe):
        with fiber_flow(pos, lengths) as (fl, dn):
            s = timestep.Stepper(fl, dn, p, ETA, tol=1e-12)
            t, dt, log = timestep.run(s, 4.5 * DT, DT, adaptive=False, observe=obs)
            results.append((t, dt, log, fl.fibers(), s.last[0].copy(), s.last[1].copy()))
    a, b = results
    assert a[:3] == b[:3]
    for k in (3, 4, 5):
        assert np.array_equal(a[k], b[k])
    assert len(seen) == sum(1 for e in a[2] if e[2]) == 5
    assert [s_[0] for s_ in seen] == [e[0] for e in a[2]]
    # free fibers in a uniform background carry next to no force: the field away from them is that background
    assert all(np.abs(v - np.array([0.3, -0.2, 0.5])).max() < 1e-6 for _, v, _ in seen)

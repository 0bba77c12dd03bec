"""GPU tests of the right-hand side of the whole system (include/skelly_b200_flow.h skb_flow_build_system_rhs / _device,
skb_mflow_build_system_rhs): System::prep_state_for_solver (system.cpp:398-458) on the device, against
tests/system_rhs_reference.py at the project's gate (1e-12 relative, max-norm and l2) per block and per body, and
bitwise against the calls it is built from.  Shapes as tests/test_gpu_system_matvec.py; the fast-path shape (>= 4096
fiber and >= 256 periphery nodes) runs with the cross kernel on and off and with the fused self-exclusion on and
off."""
import numpy as np
import pytest

import skellysim_b200 as skb
import system_rhs_reference as rr
from conftest import rel_max
from oracle.fiber_fd import compute_matrices
from skellysim_b200 import capi, distributed
from skellysim_b200.solver_hydro import SystemOperator
from test_gpu_flow import load
from test_gpu_mflow_system import device_lists, setup_mflow
from test_gpu_system_matvec import TOL, _check, blocks, make_case, setup_flow

pytestmark = pytest.mark.gpu
ETA, DT = 0.9, 1e-3
SHAPES = {"small": dict(n_fibers=30, n_shell=300, n_body_nodes=600, n_bodies=2, nodes=(8, 16, 32, 64)),
          "fast": dict(n_fibers=130, n_shell=300, n_body_nodes=400, n_bodies=2, nodes=(32,)),
          "mflow": dict(n_fibers=120, n_shell=300, n_body_nodes=600, n_bodies=3, nodes=(16, 32, 48, 64, 96))}


def rhs_case(name, seed):
    """make_case of tests/test_gpu_system_matvec.py with the reference's class matrices (the RHS uses them), per-fiber
    parameters of all four boundary-condition combinations, external forces, F_T, three point sources and a linear
    background flow"""
    fib, shell, bodies, ops, links, M, Minv, x = make_case(seed, **SHAPES[name])
    for n in set(ops["n_nodes"]):
        m = compute_matrices(n)
        ops["D_1_0"][n], ops["P"][n] = m["D_1_0"], m["P_downsample_bc"]
        ops["D_2_0"][n], ops["D_3_0"][n], ops["D_4_0"][n] = m["D_2_0"], m["D_3_0"], m["D_4_0"]
    rng = np.random.default_rng(seed + 7)
    nfib, nf = len(fib["n_nodes"]), fib["pos"].shape[0]
    lp = np.asarray(fib["lengths"]) * rng.uniform(0.95, 1.05, nfib)
    E = rng.uniform(1e-3, 1e-2, nfib)
    mc, ph = np.arange(nfib) % 2, (np.arange(nfib) // 2) % 2
    params = (lp, E, 0.0125, 500.0, 1.0, mc, ph)
    fparams = [dict(length_prev=lp[f], bending_rigidity=E[f], radius=0.0125, penalty_param=500.0, beta_tstep=1.0,
                    minus_clamped=bool(mc[f]), plus_pinned=bool(ph[f])) for f in range(nfib)]
    src = dict(f_ext=rng.uniform(-1, 1, (nf, 3)), ft=rng.uniform(-1, 1, (len(bodies["n_nodes"]), 6)),
               points=(rng.uniform(-1, 1, (3, 3)), rng.normal(size=(3, 3)), rng.normal(size=(3, 3))),
               background=([1, 0, 2], np.array([0.5, -0.25, 0.1]), np.array([0.1, 0.2, -0.3])),
               v_growth=rng.uniform(-1, 1, nfib), force_scale=rng.uniform(-2, 2, nfib))
    return fib, dict(shell, M=M, Minv=Minv), bodies, ops, links, x, params, fparams, src


def set_sources(fl, src):
    fl.set_point_sources(*src["points"])
    fl.set_background(*src["background"])


def rhs_of(fl, params, src, f_ext=True, ft=True):
    return fl.build_system_rhs(*params, DT, ETA, f_external=src["f_ext"] if f_ext else None,
                               body_forces_torques=src["ft"] if ft else None, v_growth=src["v_growth"],
                               force_scale=src["force_scale"])


def body_rows(bodies):
    off = 0
    for n in bodies["n_nodes"]:
        yield slice(off, off + 3 * n), slice(off + 3 * n, off + 3 * n + 6)
        off += 3 * n + 6


def check_rhs(got, ref, fib, shell, bodies, tol=TOL):
    """per block; per body its node rows at the gate and its six rows exactly +0.0"""
    for g, r in zip(blocks(got, fib, shell), blocks(ref, fib, shell)):
        _check(g, r, tol)
    g_b, r_b = blocks(got, fib, shell)[2], blocks(ref, fib, shell)[2]
    for nodes, six in body_rows(bodies):
        _check(g_b[nodes], r_b[nodes], tol)
        assert np.array_equal(g_b[six], np.zeros(6)) and not np.signbit(g_b[six]).any()


def reference(fib, shell, bodies, fparams, src, **kw):
    return rr.system_rhs(fib, shell, bodies, fparams, ETA, DT, f_ext=src["f_ext"], ft=src["ft"],
                         points=src["points"], background=src["background"], v_growth=src["v_growth"],
                         force_scale=src["force_scale"], **kw)[0]


@pytest.mark.parametrize("name,cross,fused", [("small", -1, 0), ("fast", 1, 0), ("fast", 0, 0), ("fast", 1, 1),
                                              ("fast", 0, 1)])
def test_rhs_matches_the_restatement(name, cross, fused):
    fib, shell, bodies, ops, links, x, params, fparams, src = rhs_case(name, 61)
    ref = reference(fib, shell, bodies, fparams, src)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        fl.set_cross(cross)
        fl.set_self_exclusion(bool(fused))
        set_sources(fl, src)
        got = rhs_of(fl, params, src)
        assert fl.stats()["launches"] > 0
    check_rhs(got, ref, fib, shell, bodies)
    # the planted count-per-member defect is visible at this gate
    bad = reference(fib, shell, bodies, fparams, src, defect="ft_twice")
    assert rel_max(blocks(bad, fib, shell)[2], blocks(got, fib, shell)[2]) > 1e3 * TOL


@pytest.mark.parametrize("name", ["small", "fast"])
def test_bitwise_identities_with_the_separate_calls(name):
    fib, shell, bodies, ops, links, x, params, fparams, src = rhs_case(name, 62)
    nf, ns, nb = fib["pos"].shape[0], shell["pos"].shape[0], bodies["pos"].shape[0]
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        got = rhs_of(fl, params, src)
        v = fl.matvec(src["f_ext"], np.zeros((ns, 3)), np.zeros((nb, 3)), src["ft"], ETA)
        fib_rhs = fl.build_fiber_rhs(*params, DT, ETA, v_on_fibers=v[:nf], f_external=src["f_ext"],
                                     v_growth=src["v_growth"], force_scale=src["force_scale"])
        zero_ft = fl.build_system_rhs(*params, DT, ETA, f_external=src["f_ext"],
                                      body_forces_torques=np.zeros_like(src["ft"]), v_growth=src["v_growth"],
                                      force_scale=src["force_scale"])
        no_ft = rhs_of(fl, params, src, ft=False)
        # no forces at all: the flow is the point sources and the background alone
        set_sources(fl, src)
        srcs = rhs_of(fl, params, src, f_ext=False, ft=False)
        r_all = np.concatenate([fib["pos"], shell["pos"], bodies["pos"]])
        vat = fl.velocity_at_targets(r_all, np.zeros((nf, 3)), np.zeros((ns, 3)), np.zeros((nb, 3)),
                                     np.zeros((len(bodies["n_nodes"]), 6)), ETA)
        fib_src = fl.build_fiber_rhs(*params, DT, ETA, v_on_fibers=vat[:nf], v_growth=src["v_growth"],
                                     force_scale=src["force_scale"])
    g_f, g_s, g_b = blocks(got, fib, shell)
    assert np.array_equal(g_f, fib_rhs)
    assert np.array_equal(g_s, -v[nf:nf + ns].reshape(-1))
    node = nf + ns
    for (nodes, six), n in zip(body_rows(bodies), bodies["n_nodes"]):
        assert np.array_equal(g_b[nodes], -v[node:node + n].reshape(-1))
        assert np.array_equal(g_b[six], np.zeros(6)) and not np.signbit(g_b[six]).any()
        node += n
    assert np.array_equal(zero_ft, no_ft)
    s_f, s_s, s_b = blocks(srcs, fib, shell)
    assert np.array_equal(s_f, fib_src)
    assert np.array_equal(s_s, -vat[nf:nf + ns].reshape(-1))
    node = nf + ns
    for (nodes, _), n in zip(body_rows(bodies), bodies["n_nodes"]):
        assert np.array_equal(s_b[nodes], -vat[node:node + n].reshape(-1))
        node += n


def test_reproducible_and_the_device_form_on_a_side_stream():
    import torch
    fib, shell, bodies, ops, links, x, params, fparams, src = rhs_case("small", 63)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        set_sources(fl, src)
        r1, r2 = rhs_of(fl, params, src), rhs_of(fl, params, src)
        d_f, d_F, d_T = t(src["f_ext"]), t(src["ft"][:, :3]), t(src["ft"][:, 3:])
        d_rhs = torch.full((fl.solution_size(),), float("nan"), dtype=torch.float64, device=dev)
        a = torch.randn(4096, 4096, device=dev)
        busy, side = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
        torch.cuda.synchronize()
        with torch.cuda.stream(busy):
            for _ in range(8):
                a = a @ a / 64.0
        fl.build_system_rhs_device(*params, DT, ETA, d_f.data_ptr(), d_F.data_ptr(), d_T.data_ptr(),
                                   d_rhs.data_ptr(), v_growth=src["v_growth"], force_scale=src["force_scale"],
                                   stream=side.cuda_stream)
        torch.cuda.synchronize()
        got = d_rhs.cpu().numpy()
    assert np.array_equal(r1, r2)
    assert np.array_equal(got, r1)


def test_the_rhs_leaves_the_operators_unchanged():
    fib, shell, bodies, ops, links, x, params, fparams, src = rhs_case("small", 64)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        r0, p0 = fl.apply_system_matvec(x, ETA, dense=dn), fl.apply_system_preconditioner(x, dense=dn)
        o0 = fl.get_fiber_operators()
        set_sources(fl, src)
        rhs_of(fl, params, src)
        assert np.array_equal(fl.apply_system_matvec(x, ETA, dense=dn), r0)
        assert np.array_equal(fl.apply_system_preconditioner(x, dense=dn), p0)
        o1 = fl.get_fiber_operators()
    for k in ("A", "force", "A_inv"):
        assert all(np.array_equal(a, b) for a, b in zip(o0[k], o1[k])), k
    assert np.array_equal(o0["xs"], o1["xs"])


def test_refusals_come_before_any_launch_and_leave_the_next_call_unchanged():
    fib, shell, bodies, ops, links, x, params, fparams, src = rhs_case("small", 65)
    nf = fib["pos"].shape[0]

    def refused(call):
        before = capi.launch_count()
        with pytest.raises(skb.SkbError, match="error 1:"):
            call()
        assert capi.launch_count() == before

    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        set_sources(fl, src)
        r0 = rhs_of(fl, params, src)
        refused(lambda: fl.build_system_rhs(*params, 0.0, ETA))                                  # dt
        refused(lambda: fl.build_system_rhs(*params, DT, -1.0))                                  # eta
        refused(lambda: fl.build_system_rhs(*(params[:2] + (0.0,) + params[3:]), DT, ETA))       # radius
        refused(lambda: fl.build_system_rhs(*(params[:5] + (2,) + params[6:]), DT, ETA))         # a flag
        refused(lambda: fl.build_system_rhs(*params, DT, ETA, v_growth=np.full(30, np.nan)))     # v_growth
        L = capi.library()
        out = np.zeros(fl.solution_size())
        refused(lambda: capi._check(L.skb_flow_build_system_rhs(fl._h, None, None, None, None, None, DT, ETA,
                                                                capi._p(out))))              # NULL params
        p = capi.fiber_params(30, *params)
        refused(lambda: capi._check(L.skb_flow_build_system_rhs(fl._h, capi._params_ptr(p), None, None, None, None,
                                                                DT, ETA, None)))              # NULL rhs
        f_bad = src["f_ext"].copy()
        f_bad[3, 1] = np.nan
        refused(lambda: fl.build_system_rhs(*params, DT, ETA, f_external=f_bad))                 # non-finite force
        ft_bad = src["ft"].copy()
        ft_bad[1, 4] = np.inf
        refused(lambda: fl.build_system_rhs(*params, DT, ETA, body_forces_torques=ft_bad))      # non-finite torque
        fl.set_target_window(0, nf)
        refused(lambda: fl.build_system_rhs(*params, DT, ETA))                                   # window
        fl.set_target_window(0, -1)
        assert np.array_equal(rhs_of(fl, params, src), r0)
        fl.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])                       # drops the operators
        refused(lambda: rhs_of(fl, params, src))
        fl.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"])
        assert np.array_equal(rhs_of(fl, params, src), r0)  # needs neither A_inv nor the links
    empty = dict(pos=np.zeros((0, 3)), normals=np.zeros((0, 3)), centers=np.zeros((0, 3)))
    with skb.Flow(0) as fl:  # a node count without its derivative matrices
        load(fl, dict(pos=fib["pos"][:8], n_nodes=[8], lengths=[1.0]), empty, empty)
        m = compute_matrices(8)
        fl.set_fiber_class(8, m["D_1_0"], m["P_downsample_bc"])
        refused(lambda: fl.build_system_rhs(1.0, 2.5e-3, 0.0125, 500.0, 1.0, 0, 0, DT, ETA))
    with skb.Flow(0) as fl:  # a group member
        load(fl, fib, shell, dict(pos=bodies["pos"], normals=bodies["normals"], centers=bodies["centers"]))
        fl.group_init(0, 2)
        refused(lambda: fl.build_system_rhs(*params, DT, ETA))


def test_gmres_on_the_device_operators_advects_free_fibers_in_a_uniform_flow():
    """Straight free fibers in a uniform background flow U, no periphery, no bodies: the exact solution of A x = b is every
    fiber advected by dt U with zero tension (its bending and tension forces vanish, so no fiber moves another).  scipy's
    GMRES runs on the host over A P^-1 (SystemOperator.apply after .apply_preconditioner, both on the device) with b =
    SystemOperator.rhs.  Bound, fixed before the run: with r = b - A x the true residual (one more device matvec) and
    cond(A) numpy's 2-norm condition number of the assembled system matrix (its columns are device matvecs),
        ||x - x*||_2 <= 4 cond(A) (||r||_2 / ||b||_2 + 64 u) ||x*||_2,   u = 2^-53,
    the perturbation bound of a linear system, with slack for the rounding of r itself."""
    import scipy.sparse.linalg as sla
    import torch
    rng = np.random.default_rng(66)
    n_fibers, n = 4, 16
    pos, lengths = [], []
    for f in range(n_fibers):
        t = rng.normal(size=3)
        t /= np.linalg.norm(t)
        L = rng.uniform(0.6, 1.2)
        pos.append(np.array([3.0 * f, 0.0, 0.0]) + np.linspace(0.0, L, n)[:, None] * t)
        lengths.append(L)
    r_fib = np.concatenate(pos)
    Uf = np.array([0.3, -0.2, 0.5])
    params = (np.array(lengths), 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)
    dev = torch.device("cuda", 0)
    with skb.Flow(0) as fl:
        fl.set_fibers(r_fib, [n] * n_fibers, lengths)
        fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_bodies(np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
        m = compute_matrices(n)
        fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
        fl.build_fiber_operators(*params, DT, ETA)
        fl.set_body_operators([], [], np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_fiber_links(None)
        fl.set_background([0, 1, 2], np.zeros(3), Uf)
        op = SystemOperator(fl, None, ETA, dev)
        b = op.rhs(params, DT).cpu().numpy()
        N = op.n
        to = lambda v: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(dev)
        A = lambda v: op.apply(to(v)).cpu().numpy()
        AP = sla.LinearOperator((N, N), matvec=lambda v: op.apply(op.apply_preconditioner(to(v))).cpu().numpy())
        z, info = sla.gmres(AP, b, rtol=1e-14, atol=0.0, restart=N, maxiter=4)
        xg = op.apply_preconditioner(to(z)).cpu().numpy()
        r = b - A(xg)
        Afull = np.stack([A(e) for e in np.eye(N)], axis=1)
    x_star = np.concatenate([np.concatenate([(p + DT * Uf).T.reshape(-1), np.zeros(n)]) for p in pos])
    cond = np.linalg.cond(Afull)
    bound = 4 * cond * (np.linalg.norm(r) / np.linalg.norm(b) + 64 * 2.0 ** -53) * np.linalg.norm(x_star)
    err = np.linalg.norm(xg - x_star)
    print(f"\ngmres info {info}, |r|/|b| {np.linalg.norm(r) / np.linalg.norm(b):.1e}, cond {cond:.1e}, "
          f"error {err:.1e}, bound {bound:.1e}")
    assert err <= bound, (err, bound)


def _mflow_rhs(mf, params, src):
    return mf.build_system_rhs(*params, DT, ETA, f_external=src["f_ext"], body_forces_torques=src["ft"],
                               v_growth=src["v_growth"], force_scale=src["force_scale"])


@pytest.mark.parametrize("cross", [0, 1])
def test_mflow_rhs_matches_the_single_device_and_the_restatement(cross):
    fib, shell, bodies, ops, links, x, params, fparams, src = rhs_case("mflow", 67)
    ref = reference(fib, shell, bodies, fparams, src)
    rng = np.random.default_rng(5)
    r_trg = rng.uniform(-2, 2, (300, 3))
    nf, ns, nb = fib["pos"].shape[0], shell["pos"].shape[0], bodies["pos"].shape[0]
    strengths = (rng.uniform(-1, 1, (nf, 3)), rng.uniform(-1, 1, (ns, 3)), rng.uniform(-1, 1, (nb, 3)),
                 rng.uniform(-1, 1, (len(bodies["n_nodes"]), 6)))
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        fl.set_cross(cross)
        set_sources(fl, src)
        single = rhs_of(fl, params, src)
        vat = fl.velocity_at_targets(r_trg, *strengths, ETA)
    check_rhs(single, ref, fib, shell, bodies)
    for devs in device_lists():
        with skb.MultiFlow(devs) as mf:
            mf.set_cross(cross)
            setup_mflow(mf, fib, shell, bodies, ops, links)
            mf.set_point_sources(*src["points"])
            mf.set_background(*src["background"])
            got = _mflow_rhs(mf, params, src)
            again = _mflow_rhs(mf, params, src)
            out = np.full(mf.solution_size(), np.nan)  # every row is written by its owner
            p = capi.fiber_params(len(fib["n_nodes"]), *params)
            capi._check(capi.library().skb_mflow_build_system_rhs(
                mf._h, capi._params_ptr(p), capi._p(src["v_growth"]), capi._p(src["force_scale"]),
                capi._p(np.ascontiguousarray(src["f_ext"])), capi._p(np.ascontiguousarray(src["ft"])), DT, ETA,
                capi._p(out)))
            parts = [mf.partition(g) for g in range(len(devs))]
            mvat = mf.velocity_at_targets(r_trg, *strengths, ETA)
        assert np.array_equal(got, again), devs
        assert np.array_equal(out, got), devs
        owned = np.concatenate([distributed.system_rows(pt, fib["n_nodes"], ns, bodies["n_nodes"]) for pt in parts])
        assert np.array_equal(np.sort(owned), np.arange(got.size)), devs  # one owner per row
        if len(devs) == 1:
            assert np.array_equal(got, single)
        check_rhs(got, single, fib, shell, bodies)
        check_rhs(got, ref, fib, shell, bodies)  # F_T counted once, however many members
        _check(mvat, vat)

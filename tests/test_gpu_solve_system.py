"""GPU tests of the whole-system solve (include/skelly_b200_flow.h skb_flow_set_gmres, skb_flow_solve_system / _device,
SystemOperator.solve): Solver::solve (solver_hydro.cpp:64-95) on the device, against tests/gmres_reference.py fed the
device's own operators, against two physical closed forms, and on its restarts, limits, refusals and reproducibility.

The systems are make_case / edge_case's (tests/test_gpu_system_matvec.py, tests/test_gpu_system_edges.py) with
preconditioners that are the exact block inverses -- the fibers' A_^-1, M_inv = inv(M) for a well-conditioned M, the
bodies' A_^-1 -- so A P^-1 is I plus the hydrodynamic couplings and GMRES converges in tens of steps.

HISTORY_BOUND: the device's implicit relative residual after every step stays within this of the restatement's.  It is
10x the worst |rho_1(k) - rho_2(k)| / ||b|| seen on the CPU between two runs of the restatement on these systems (with
system_reference.py's operators), one with numpy's dots and one with the dots summed in the kernels' blocked order
(gmres_reference.blocked_dot), over every system a test below compares with the restatement (CALIBRATED) at tol
1e-10: worst 1.22e-15 (FPB of seed 72 with 3 blocks; 5.6e-17 or less elsewhere).  tests/test_solve_calibration_cpu.py
recomputes it and holds each case below HISTORY_BOUND / 10."""
import contextlib

import numpy as np
import pytest

import gmres_reference as gr
import skellysim_b200 as skb
from oracle.fiber_fd import compute_matrices
from skellysim_b200 import capi
from skellysim_b200.solver_hydro import SystemOperator
from test_gpu_system_edges import host_body_solve, sphere
from test_gpu_system_edges import edge_case
from test_gpu_system_matvec import setup_flow

pytestmark = pytest.mark.gpu
ETA, DT, TOL = 0.9, 1e-3, 1e-10
HISTORY_BOUND = 1.22e-14

# make_case keywords: fibers of 8..64 nodes in a periphery (and two bodies), the fast-path shape (symmetric and cross
# kernels, background streamer: >= 4096 fiber and >= 256 periphery nodes) and shapes with an empty block.  The bodies
# take their true singularity-subtraction vectors and operator (system_reference.body_operator), so that their inverse
# is the exact block inverse; make_case's random ones are no preconditioner for the body block the device applies
SHAPES = {"FP": dict(n_fibers=30, n_shell=300, n_body_nodes=0, n_bodies=0),
          "FPB": dict(n_fibers=30, n_shell=300, n_body_nodes=400, n_bodies=2, bound=False),
          "fast": dict(n_fibers=150, n_shell=500, n_body_nodes=0, n_bodies=0, nodes=(32,)),
          "F": dict(n_fibers=30, n_shell=0, n_body_nodes=0, n_bodies=0),
          "P": dict(n_fibers=0, n_shell=300, n_body_nodes=0, n_bodies=0)}
# M1 and M5 of tests/test_gpu_system_edges.py: on three members the middle one of M1 owns no fiber and the last one of
# M5 owns nothing at all; FPB: every block on every member
MEMBER_SHAPES = {"M1": dict(n_fibers=2, n_shell=300, n_body_nodes=600, n_bodies=2, bound=False),
                 "M5": dict(n_fibers=0, n_shell=2, n_body_nodes=2, n_bodies=1),
                 "FPB": SHAPES["FPB"]}
# (shape, seed, shape keywords, num_blocks) of every comparison with the restatement below
CALIBRATED = ([(name, 71, None, 300) for name in SHAPES] + [("FPB", 72, None, 3)]
              + [(name, 5, kw, 300) for name, kw in MEMBER_SHAPES.items()])
COUPLING = 1e-2  # make_case's random force operators scaled: the fibers' flow on each other a perturbation of A_


def solve_case(name, seed=71, shape=None):
    """edge_case on the shape with a well-conditioned M and its exact inverse; x the solution of the tests' b = A x"""
    fib, shell, bodies, ops, links, x, params, fparams, src = edge_case(shape or SHAPES[name], seed, rhs=False)
    ops["force"] = [COUPLING * F for F in ops["force"]]
    bodies = true_bodies(bodies)
    ns = shell["pos"].shape[0]
    rng = np.random.default_rng(seed + 3)
    M = np.eye(3 * ns) + 0.1 * rng.normal(size=(3 * ns, 3 * ns)) / np.sqrt(max(3 * ns, 1))
    shell = dict(shell, M=M, Minv=np.linalg.inv(M))
    return fib, shell, bodies, ops, links, x


def true_bodies(bodies):
    """bodies with ex / ey / ez and A of update_singularity_subtraction_vecs / body_operator at their own nodes"""
    import system_reference as sr
    off, ex, ey, ez, A = 0, [], [], [], []
    for b, n in enumerate(bodies["n_nodes"]):
        sl = slice(off, off + n)
        off += n
        r, nrm, w = bodies["pos"][sl], bodies["normals"][sl], bodies["weights"][sl]
        e = sr.singularity_vectors(r, nrm, w)
        ex.append(e[0]), ey.append(e[1]), ez.append(e[2])
        A.append(sr.body_operator(r, nrm, bodies["centers"][b], w, *e))
    cat = lambda parts: np.concatenate(parts) if parts else np.zeros((0, 3))
    return dict(bodies, ex=cat(ex), ey=cat(ey), ez=cat(ez), A=A)


@contextlib.contextmanager
def flow_of(fib, shell, bodies, ops, links):
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0])) if shell["pos"].shape[0] else None
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        yield fl, dn


def _torch():
    import torch
    return torch, torch.device("cuda", 0)


def operators(op):
    """A and P^-1 of the device as numpy callables (for the restatement)"""
    torch, dev = _torch()
    to = lambda v: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(dev)
    return (lambda v: op.apply(to(v)).cpu().numpy()), (lambda v: op.apply_preconditioner(to(v)).cpu().numpy())


def against_restatement(hist, info, ref_info, tol, b_norm):
    """the history within HISTORY_BOUND step by step, the iteration count equal -- or one apart only where the
    restatement's deciding estimate lies within the bound of tol"""
    k = min(len(hist), len(ref_info["history"]))
    d = np.abs(hist[:k] - ref_info["history"][:k])
    assert d.max() <= HISTORY_BOUND, (d.max(), int(d.argmax()))
    if info["iterations"] != ref_info["iterations"]:
        assert abs(info["iterations"] - ref_info["iterations"]) == 1, (info, ref_info)
        near = ref_info["history"][min(info["iterations"], ref_info["iterations"]):][:2]
        assert np.abs(near - tol).min() <= HISTORY_BOUND, (near, tol)


@pytest.mark.parametrize("name", list(SHAPES))
def test_solve_matches_the_restatement(name):
    torch, dev = _torch()
    fib, shell, bodies, ops, links, x_true = solve_case(name)
    with flow_of(fib, shell, bodies, ops, links) as (fl, dn):
        op = SystemOperator(fl, dn, ETA, dev)
        b = op.apply(torch.from_numpy(x_true).to(dev)).clone()
        x, info = op.solve(b, tol=TOL)
        launches = op.launches
        x_np, b_np = x.cpu().numpy(), b.cpu().numpy()
        A, P = operators(op)
        r_host = np.linalg.norm(b_np - A(x_np))
        _, ref = gr.gmres(A, P, b_np, tol=TOL)
    print(f"\n{name}: n {b_np.size}, {info['iterations']} steps (restatement {ref['iterations']}), "
          f"explicit {info['explicit_residual']:.2e}, |x - x*| / |x*| "
          f"{np.linalg.norm(x_np - x_true) / np.linalg.norm(x_true):.1e}")
    assert info["converged"] == 1 and info["restarts"] == 0
    assert 1 <= info["iterations"] <= 100
    assert launches > 3 * info["iterations"]  # the flow's stats count the solve's launches
    assert info["explicit_residual"] <= TOL and info["implicit_residual"] <= TOL
    assert info["residual"] == pytest.approx(r_host, rel=1e-9)
    assert len(info["history"]) == info["iterations"] + 1 and info["history"][0] == 1.0
    against_restatement(info["history"], info, ref, TOL, np.linalg.norm(b_np))


def test_restarts_and_limits():
    torch, dev = _torch()
    fib, shell, bodies, ops, links, x_true = solve_case("FPB", 72)
    with flow_of(fib, shell, bodies, ops, links) as (fl, dn):
        op = SystemOperator(fl, dn, ETA, dev)
        b = op.apply(torch.from_numpy(x_true).to(dev)).clone()
        A, P = operators(op)
        b_np = b.cpu().numpy()
        x5, i5 = op.solve(b, tol=TOL, num_blocks=3)
        _, r5 = gr.gmres(A, P, b_np, tol=TOL, num_blocks=3)
        xs, ishort = op.solve(b, tol=TOL, max_iters=3)
        _, rshort = gr.gmres(A, P, b_np, tol=TOL, max_iters=3)
        z, iz = op.solve(torch.zeros_like(b), tol=TOL)
        z = z.cpu().numpy()
    assert i5["converged"] and i5["restarts"] >= 2 and i5["explicit_residual"] <= TOL, i5
    against_restatement(i5["history"], i5, r5, TOL, np.linalg.norm(b_np))
    assert ishort["converged"] == 0 and ishort["iterations"] == 3 and rshort["iterations"] == 3
    assert abs(ishort["explicit_residual"] - rshort["explicit_residual"]) <= 1e-12
    assert np.array_equal(z, np.zeros_like(z)) and iz["converged"] == 1 and iz["iterations"] == 0
    assert iz["residual"] == 0.0


def test_the_empty_system():
    torch, dev = _torch()
    empty = np.zeros((0, 3))
    with skb.Flow(0) as fl:
        fl.set_fibers(empty, [], [])
        fl.set_periphery(empty, empty)
        fl.set_bodies(empty, empty, empty)
        before = capi.launch_count()
        x, info, hist = fl.solve_system(np.zeros(0), ETA)  # no workspace needed
        assert capi.launch_count() == before
        fl.set_gmres(300)  # and one of size 0 is fine
        op = SystemOperator(fl, None, ETA, dev)
        xs, infos = op.solve(torch.zeros(0, dtype=torch.float64, device=dev))
        assert capi.launch_count() == before
    assert x.size == 0 and info["converged"] == 1 and info["iterations"] == 0
    assert xs.numel() == 0 and infos["converged"] == 1 and infos["iterations"] == 0


def test_refusals_leave_x_untouched_and_launch_nothing():
    torch, dev = _torch()
    fib, shell, bodies, ops, links, x_true = solve_case(
        "FB", 73, shape=dict(n_fibers=30, n_shell=300, n_body_nodes=600, n_bodies=2))
    L = capi.library()
    with flow_of(fib, shell, bodies, ops, links) as (fl, dn):
        n = fl.solution_size()
        d_b = torch.from_numpy(x_true).to(dev)
        d_x = torch.full((n,), float("nan"), dtype=torch.float64, device=dev)

        def refused(call):
            before = capi.launch_count()
            with pytest.raises(skb.SkbError, match="error 1:"):
                call()
            torch.cuda.synchronize()
            assert capi.launch_count() == before
            assert torch.isnan(d_x).all()

        solve = lambda **kw: fl.solve_system_device(kw.pop("dense", dn), d_b.data_ptr(), kw.pop("eta", ETA),
                                                    d_x.data_ptr(), **kw)
        refused(lambda: solve(num_blocks=10))                         # no skb_flow_set_gmres
        fl.set_gmres(20)
        refused(lambda: solve(num_blocks=21))                         # beyond the workspace
        refused(lambda: solve(num_blocks=0))
        refused(lambda: solve(num_blocks=capi.GMRES_MAX_BLOCKS + 1))
        refused(lambda: solve(num_blocks=10, tol=0.0))
        refused(lambda: solve(num_blocks=10, tol=-1e-10))
        refused(lambda: solve(num_blocks=10, tol=float("nan")))
        refused(lambda: solve(num_blocks=10, tol=float("inf")))
        refused(lambda: solve(num_blocks=10, max_iters=-1))
        refused(lambda: solve(num_blocks=10, eta=0.0))
        refused(lambda: solve(num_blocks=10, dense=None))             # the periphery needs its operators
        refused(lambda: capi._check(L.skb_flow_solve_system_device(fl._h, dn._h, None, ETA, TOL, 10, 10, None,
                                                                   None, None, None)))  # NULL info
        refused(lambda: capi._check(L.skb_flow_set_gmres(fl._h, 0)))
        fl.set_fiber_links(None)  # fibers and bodies without links: fine for the matvec (no fiber bound)
        fl.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])  # drops the body operators
        refused(lambda: solve(num_blocks=10))
        fl.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"])
        refused(lambda: solve(num_blocks=10))                         # no body A_inv: no preconditioner
        fl.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"],
                              [np.linalg.inv(A) for A in bodies["A"]])
        fl.set_fiber_links(links["body"], links["site"], links["rigidity"])
        info, _ = solve(num_blocks=10, max_iters=2)                   # and now it runs
        torch.cuda.synchronize()
        assert info["iterations"] == 2 and not torch.isnan(d_x).any()
        d_x.fill_(float("nan"))
        last = int(fib["n_nodes"][-1])
        fl.set_fibers(fib["pos"][:-last], fib["n_nodes"][:-1], fib["lengths"][:-1])  # a new solution size
        refused(lambda: solve(num_blocks=10))


def test_reproducible_and_the_device_form_on_a_side_stream():
    torch, dev = _torch()
    fib, shell, bodies, ops, links, x_true = solve_case("fast", 74)
    with flow_of(fib, shell, bodies, ops, links) as (fl, dn):
        fl.set_gmres(300)
        b = fl.apply_system_matvec(x_true, ETA, dense=dn)
        x1, i1, h1 = fl.solve_system(b, ETA, dense=dn, tol=TOL)
        x2, i2, h2 = fl.solve_system(b, ETA, dense=dn, tol=TOL)
        d_b = torch.from_numpy(b).to(dev)
        d_x = torch.full_like(d_b, float("nan"))
        a = torch.randn(4096, 4096, device=dev)
        busy, side = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
        torch.cuda.synchronize()
        with torch.cuda.stream(busy):
            for _ in range(8):
                a = a @ a / 64.0
        i3, h3 = fl.solve_system_device(dn, d_b.data_ptr(), ETA, d_x.data_ptr(), tol=TOL, stream=side.cuda_stream)
        torch.cuda.synchronize()
        x3 = d_x.cpu().numpy()
    assert i1["converged"] and i1 == i2 and i1 == i3
    assert np.array_equal(x1, x2) and np.array_equal(x1, x3)
    assert np.array_equal(h1, h2) and np.array_equal(h1, h3)


def test_free_fibers_in_a_uniform_flow_advect_with_zero_tension():
    """Straight free fibers in a uniform background flow U, no periphery, no bodies, fiber operators and their inverse
    built on the device and the RHS too: the exact solution is every fiber advected by dt U with zero tension.  Bound
    (tests/test_gpu_system_rhs.py's, with the solve's own explicit residual): ||x - x*|| <= 4 cond(A) (||r|| / ||b|| +
    64 u) ||x*||."""
    torch, dev = _torch()
    rng = np.random.default_rng(66)
    n_fibers, n = 4, 16
    pos, lengths = [], []
    for f in range(n_fibers):
        t = rng.normal(size=3)
        t /= np.linalg.norm(t)
        L = rng.uniform(0.6, 1.2)
        pos.append(np.array([3.0 * f, 0.0, 0.0]) + np.linspace(0.0, L, n)[:, None] * t)
        lengths.append(L)
    Uf = np.array([0.3, -0.2, 0.5])
    params = (np.array(lengths), 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)
    with skb.Flow(0) as fl:
        fl.set_fibers(np.concatenate(pos), [n] * n_fibers, lengths)
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
        b = op.rhs(params, DT)
        x, info = op.solve(b, tol=1e-14)
        x = x.cpu().numpy()
        A = operators(op)[0]
        Afull = np.stack([A(e) for e in np.eye(op.n)], axis=1)
    x_star = np.concatenate([np.concatenate([(p + DT * Uf).T.reshape(-1), np.zeros(n)]) for p in pos])
    cond = np.linalg.cond(Afull)
    bound = 4 * cond * (info["explicit_residual"] + 64 * 2.0 ** -53) * np.linalg.norm(x_star)
    err = np.linalg.norm(x - x_star)
    print(f"\n{info['iterations']} steps, explicit {info['explicit_residual']:.1e}, cond {cond:.1e}, error {err:.1e}, "
          f"bound {bound:.1e}")
    assert info["converged"] and err <= bound, (err, bound, info)


def test_a_sphere_moves_by_stokes_law_and_turns_by_its_rotlet():
    """test_gpu_system_edges.py's lone 400-node sphere with its bounds, solved by the device GMRES"""
    torch, dev = _torch()
    import system_reference as sr

    def device_solve(n, R, eta, F, L, rtol):
        r, nrm, w = sphere(n, R)
        ex, ey, ez = sr.singularity_vectors(r, nrm, w)
        A = sr.body_operator(r, nrm, np.zeros(3), w, ex, ey, ez)
        to = lambda v: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(dev)
        with skb.Flow(0) as fl:
            fl.set_fibers(np.zeros((0, 3)), [], [])
            fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
            fl.set_bodies(r, nrm, np.zeros((1, 3)))
            fl.set_body_operators([n], w, ex, ey, ez, [np.linalg.inv(A)])
            op = SystemOperator(fl, None, eta, dev)
            b = op.rhs((1.0, 2.5e-3, 0.0125, 500.0, 1.0, 0, 0), DT, body_forces=to(np.reshape(F, (1, 3))),
                       body_torques=to(np.reshape(L, (1, 3))))
            x, info = op.solve(b, tol=rtol, num_blocks=200)
            assert info["converged"], info
            return x.cpu().numpy()

    n, rtol = 400, 1e-13
    R, eta, F = 1.0, 1.0, np.array([0.3, -0.7, 0.2])
    A, x_host = host_body_solve(n, R, eta, F, np.zeros(3))
    x_dev = device_solve(n, R, eta, F, np.zeros(3), rtol)
    cond = np.linalg.cond(A)
    err_sys = np.linalg.norm(x_dev - x_host) / np.linalg.norm(x_host)
    assert err_sys <= 4 * rtol * cond, (err_sys, cond)
    U_stokes = F / (6 * np.pi * eta * R)
    e_host = np.linalg.norm(x_host[3 * n:3 * n + 3] - U_stokes) / np.linalg.norm(U_stokes)
    e_dev = np.linalg.norm(x_dev[3 * n:3 * n + 3] - U_stokes) / np.linalg.norm(U_stokes)
    assert e_dev <= 2 * e_host, (e_dev, e_host)
    R, eta, L = 0.5, 0.7, np.array([0.2, 0.5, -0.4])
    x_rot = device_solve(n, R, eta, np.zeros(3), L, rtol)
    W = L / (8 * np.pi * eta * R ** 3)
    e_rot = np.linalg.norm(x_rot[3 * n + 3:] - W) / np.linalg.norm(W)
    assert e_rot <= 1e-12 + rtol, e_rot


# ---- members: skb_mflow and one rank per GPU -----------------------------------------------------------------------


def member_lists():
    n = capi.device_count()
    return [[0], [0, 0], [0, 0, 0]] + [list(range(k)) for k in (2, 3) if n >= k]


@pytest.mark.parametrize("name", list(MEMBER_SHAPES))
def test_members_solve_as_one_device(name):
    """skb_mflow on [0] is bitwise the single device; on several members every step stays within HISTORY_BOUND of the
    single device's restatement, and every member reports bitwise the same info and history (skb_mflow refuses
    otherwise); rank-per-GPU members (threads) are bitwise skb_mflow on the same device list, and no flag wait timed
    out"""
    from test_gpu_group_system import Members, run_all
    from test_gpu_system_edges import setup_mflow_edges
    torch, dev = _torch()
    fib, shell, bodies, ops, links, x_true = solve_case(name, 5, shape=MEMBER_SHAPES[name])
    with flow_of(fib, shell, bodies, ops, links) as (fl, dn):
        fl.set_gmres(300)
        b = fl.apply_system_matvec(x_true, ETA, dense=dn)
        x1, i1, h1 = fl.solve_system(b, ETA, dense=dn, tol=TOL)
        op = SystemOperator(fl, dn, ETA, dev)
        A, P = operators(op)
        _, ref = gr.gmres(A, P, b, tol=TOL)
    assert i1["converged"]
    for devs in member_lists():
        with skb.MultiFlow(devs) as mf:
            setup_mflow_edges(mf, fib, shell, bodies, ops, links)
            mf.set_gmres(300)
            xm, im, hm = mf.solve_system(b, ETA, tol=TOL)
            xm2, im2, hm2 = mf.solve_system(b, ETA, tol=TOL)
        assert np.array_equal(xm, xm2) and im == im2 and np.array_equal(hm, hm2), devs
        if len(devs) == 1:
            assert np.array_equal(xm, x1) and im == i1 and np.array_equal(hm, h1)
            continue
        assert im["converged"] and im["explicit_residual"] <= TOL, (devs, im)
        against_restatement(hm, im, ref, TOL, np.linalg.norm(b))
        mem = Members(devs, fib, shell, bodies, ops, links)
        try:
            for f in mem.flows:
                f.set_gmres(300)
            mem.scatter(b)
            infos, hists = [None] * mem.n, [None] * mem.n

            def solve(g):
                st = mem.streams[g]
                infos[g], hists[g] = mem.flows[g].group_solve_system_device(
                    mem.dense[g], mem.dense[g], mem.x[g].data_ptr(), ETA, mem.y[g].data_ptr(), tol=TOL,
                    stream=st.cuda_stream)
                st.synchronize()
            run_all(mem.n, solve)
            xr = mem.gather()
            missing = [f.group_error() for f in mem.flows]
        finally:
            mem.close()
        assert all(i == infos[0] for i in infos) and all(np.array_equal(h, hists[0]) for h in hists), devs
        assert infos[0] == im and np.array_equal(hists[0], hm), devs
        assert np.array_equal(xr, xm), devs
        assert all(m == -1 for m in missing), missing

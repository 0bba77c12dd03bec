"""GPU tests of the whole-vector operator and preconditioner (include/skelly_b200_flow.h skb_flow_apply_system_matvec /
_preconditioner): System::apply_matvec (system.cpp:269-324) and ::apply_preconditioner (:248-262) with the body block
and the fiber-body links on the device, against tests/system_reference.py.  Tolerance 1e-12 relative per block
(max-norm and l2), the project's parity gate."""
import numpy as np
import pytest

import skellysim_b200 as skb
import system_reference as sr
from conftest import rel_l2, rel_max
from oracle.fiber_fd import compute_matrices
from skellysim_b200.solver_hydro import SystemOperator, iterate_system
from test_gpu_fiberops import make_ops
from test_gpu_flow import load, make_system

pytestmark = pytest.mark.gpu
TOL = 1e-12
ETA = 0.9


def _check(u, ref, tol=TOL):
    assert np.isfinite(u).all()
    if ref.size == 0:
        return
    assert rel_max(u, ref) <= tol, rel_max(u, ref)
    assert rel_l2(u, ref) <= tol, rel_l2(u, ref)


def make_case(seed, n_fibers=30, n_shell=500, n_body_nodes=600, n_bodies=2, bound=True, nodes=(8, 16, 32, 64)):
    """fibers of 8..64 nodes, every other one bound to one of the bodies (free ones interleaved), 300 nodes per body,
    a periphery with random dense operators; random fiber / body operators (the kernels are linear algebra)"""
    fib, shell, body = make_system(seed, n_fibers, n_shell, n_body_nodes, n_bodies, nodes=nodes)
    rng = np.random.default_rng(seed + 100)
    ops = make_ops(fib, seed + 1)
    ops["A"] = [np.eye(4 * n) + 0.1 * A for n, A in zip(ops["n_nodes"], ops["A"])]
    ops["D_2_0"], ops["D_3_0"], ops["D_4_0"] = ({n: rng.normal(size=(n, n)) for n in ops["D_1_0"]} for _ in range(3))
    per = n_body_nodes // max(n_bodies, 1)
    nb = body["pos"].shape[0]
    bodies = dict(pos=body["pos"], normals=body["normals"], centers=body["centers"], n_nodes=[per] * n_bodies,
                  weights=rng.uniform(0.5, 1.5, nb), ex=rng.normal(size=(nb, 3)), ey=rng.normal(size=(nb, 3)),
                  ez=rng.normal(size=(nb, 3)))
    bodies["A"] = [np.eye(3 * per + 6) + 0.1 * rng.normal(size=(3 * per + 6,) * 2) / np.sqrt(3 * per) for _ in
                   range(n_bodies)]
    body_of = np.array([(f // 2) % n_bodies if (bound and n_bodies and f % 2 == 0) else -1 for f in range(n_fibers)])
    site = np.array([body["centers"][b] + 0.4 * rng.normal(size=3) if b >= 0 else rng.normal(size=3)
                     for b in body_of]).reshape(-1, 3)
    links = dict(body=body_of, site=site, rigidity=rng.uniform(0.5, 2.0, n_fibers))
    ns = shell["pos"].shape[0]
    M = rng.normal(size=(3 * ns, 3 * ns)) / np.sqrt(3 * ns)
    Minv = np.eye(3 * ns) + 0.1 * rng.normal(size=(3 * ns, 3 * ns)) / np.sqrt(3 * ns)
    n_sol = 4 * fib["pos"].shape[0] + 3 * ns + sum(3 * n + 6 for n in bodies["n_nodes"])
    x = rng.normal(size=n_sol)
    return fib, shell, bodies, ops, links, M, Minv, x


def setup_flow(fl, dn, fib, shell, bodies, ops, links, build=None):
    load(fl, fib, shell, dict(pos=bodies["pos"], normals=bodies["normals"], centers=bodies["centers"]))
    for n in ops["D_1_0"]:
        fl.set_fiber_class(n, ops["D_1_0"][n], ops["P"][n])
        if n in ops["D_2_0"]:  # (a class beyond the device build's node counts has none)
            fl.set_fiber_class_derivatives(n, ops["D_2_0"][n], ops["D_3_0"][n], ops["D_4_0"][n])
    if build is None:
        fl.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
        fl.set_fiber_preconditioner(ops["A_inv"] if "A_inv" in ops else [np.linalg.inv(A) for A in ops["A"]])
    else:
        fl.build_fiber_operators(*build)
    if bodies["n_nodes"]:
        fl.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"],
                              [np.linalg.inv(A) for A in bodies["A"]])
    else:
        fl.set_body_operators([], [], np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
    fl.set_fiber_links(links["body"], links["site"], links["rigidity"])
    if dn is not None and shell["pos"].shape[0]:
        dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, shell["M"])
        dn.set_matrix(skb.DENSE_M_INV, shell["Minv"])


def blocks(v, fib, shell):
    nf, ns = fib["pos"].shape[0], shell["pos"].shape[0]
    return v[:4 * nf], v[4 * nf:4 * nf + 3 * ns], v[4 * nf + 3 * ns:]


@pytest.mark.parametrize("operators", ["uploaded", "built"])
def test_system_matvec_matches_the_reference_block_by_block(operators):
    nodes = (8, 16, 32, 64) if operators == "uploaded" else (16, 32)
    fib, shell, bodies, ops, links, M, Minv, x = make_case(31, nodes=nodes)
    shell = dict(shell, M=M, Minv=Minv)
    build = None
    if operators == "built":
        for n in set(ops["n_nodes"]):  # the build needs the reference's class matrices
            m = compute_matrices(n)
            ops["D_1_0"][n], ops["P"][n] = m["D_1_0"], m["P_downsample_bc"]
            ops["D_2_0"][n], ops["D_3_0"][n], ops["D_4_0"][n] = m["D_2_0"], m["D_3_0"], m["D_4_0"]
        nfib = len(ops["n_nodes"])
        lp = np.asarray(fib["lengths"]) * 1.01
        build = (lp, 0.02, 0.0125, 500.0, 1.0, np.arange(nfib) % 2, (np.arange(nfib) // 2) % 2, 1e-3, ETA)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links, build)
        if build is not None:
            got = fl.get_fiber_operators(inverse=False)
            ops["A"], ops["force"], ops["xs"] = got["A"], got["force"], got["xs"]
            ops["length_prev"], ops["plus"] = list(build[0]), list(build[6])
        res = fl.apply_system_matvec(x, ETA, dense=dn)
        assert fl.stats()["launches"] > 0
    ref, vel, ft = sr.system_apply_matvec(fib, shell, bodies, ops, links, M, x, ETA)
    assert np.count_nonzero(ft) > 0 and np.count_nonzero(vel) > 0  # the links act
    for got_b, ref_b in zip(blocks(res, fib, shell), blocks(ref, fib, shell)):
        _check(got_b, ref_b)


def test_bodies_without_bound_fibers_take_the_existing_path():
    import torch
    fib, shell, bodies, ops, links, M, Minv, x = make_case(32, bound=False)
    shell = dict(shell, M=M, Minv=Minv)
    nf, ns, nb = fib["pos"].shape[0], shell["pos"].shape[0], bodies["pos"].shape[0]
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        fl.set_fiber_links(None)
        d_x, d_res = t(x), torch.zeros(x.size, dtype=torch.float64, device=dev)
        fl.apply_system_matvec_device(dn, d_x.data_ptr(), ETA, d_res.data_ptr())
        x_f, x_s, x_b = blocks(x, fib, shell)
        dens = np.concatenate([x_b[b * (3 * 300 + 6):b * (3 * 300 + 6) + 900].reshape(300, 3) for b in range(2)])
        zeros = t(np.zeros((2, 3)))
        r_f, r_s, v_b = (torch.zeros(k, dtype=torch.float64, device=dev) for k in (4 * nf, 3 * ns, 3 * nb))
        d_xf, d_xs, d_dens = t(x_f), t(x_s), t(dens)
        fl.apply_matvec_device(dn, d_xf.data_ptr(), d_xs.data_ptr(), d_dens.data_ptr(), zeros.data_ptr(),
                               zeros.data_ptr(), 0, ETA, r_f.data_ptr(), r_s.data_ptr(), v_b.data_ptr())
        torch.cuda.synchronize()
        res, r_f, r_s, v_b = (a.cpu().numpy() for a in (d_res, r_f, r_s, v_b))
    g_f, g_s, g_b = blocks(res, fib, shell)
    assert np.array_equal(g_f, r_f) and np.array_equal(g_s, r_s)
    _check(g_b, sr.body_matvec(bodies, v_b.reshape(nb, 3), x_b))


def test_system_preconditioner():
    import torch
    fib, shell, bodies, ops, links, M, Minv, x = make_case(33)
    shell = dict(shell, M=M, Minv=Minv)
    nf, ns = fib["pos"].shape[0], shell["pos"].shape[0]
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        y = fl.apply_system_preconditioner(x, dense=dn)
        x_f, x_s, x_b = blocks(x, fib, shell)
        d_xf, d_xs = t(x_f), t(x_s)
        y_f, y_s = torch.zeros_like(d_xf), torch.zeros_like(d_xs)
        fl.apply_fiber_preconditioner_device(d_xf.data_ptr(), y_f.data_ptr())
        dn.apply_device(skb.DENSE_M_INV, d_xs.data_ptr(), 0, y_s.data_ptr())
        torch.cuda.synchronize()
        y_f, y_s = y_f.cpu().numpy(), y_s.cpu().numpy()
    g_f, g_s, g_b = blocks(y, fib, shell)
    assert np.array_equal(g_f, y_f) and np.array_equal(g_s, y_s)
    m = 3 * 300 + 6
    ref_b = np.concatenate([np.linalg.inv(A) @ x_b[b * m:(b + 1) * m] for b, A in enumerate(bodies["A"])])
    _check(g_b, ref_b)


def test_isolated_body_preconditioner_inverts_the_matvec():
    from test_body_block_cpu import bodies_of
    bodies = bodies_of((200,), seed=7)
    A = sr.body_operator(bodies["pos"], bodies["normals"], bodies["centers"][0], bodies["weights"], bodies["ex"],
                         bodies["ey"], bodies["ez"])
    A_inv = np.linalg.inv(A)
    x = np.random.default_rng(8).normal(size=A.shape[0])
    err_np = np.abs(A_inv @ (A @ x) - x).max()
    empty = dict(pos=np.zeros((0, 3)), n_nodes=[], lengths=[])
    with skb.Flow(0) as fl:
        fl.set_fibers(empty["pos"], [], [])
        fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])
        fl.set_fiber_operators([], [], np.zeros((0, 3)), [], [])
        fl.set_fiber_preconditioner([])
        fl.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"], [A_inv])
        fl.set_fiber_links(None)
        ax = fl.apply_system_matvec(x, ETA)
        px = fl.apply_system_preconditioner(ax)
    _check(ax, A @ x)
    assert np.abs(px - x).max() <= 32 * err_np, (np.abs(px - x).max(), err_np)


def test_reproducible_host_device_and_input_untouched():
    import torch
    fib, shell, bodies, ops, links, M, Minv, x = make_case(34)
    shell = dict(shell, M=M, Minv=Minv)
    dev = torch.device("cuda", 0)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        x0 = x.copy()
        r1 = fl.apply_system_matvec(x, ETA, dense=dn)
        r2 = fl.apply_system_matvec(x, ETA, dense=dn)
        p1 = fl.apply_system_preconditioner(x, dense=dn)
        d_x = torch.from_numpy(x).to(dev)
        d_r, d_p = torch.zeros_like(d_x), torch.zeros_like(d_x)
        fl.apply_system_matvec_device(dn, d_x.data_ptr(), ETA, d_r.data_ptr())
        fl.apply_system_preconditioner_device(dn, d_x.data_ptr(), d_p.data_ptr())
        torch.cuda.synchronize()
        assert np.array_equal(d_x.cpu().numpy(), x0)
    assert np.array_equal(x, x0)
    assert np.array_equal(r1, r2)
    assert np.array_equal(d_r.cpu().numpy(), r1) and np.array_equal(d_p.cpu().numpy(), p1)


def _refused(call):
    with pytest.raises(skb.SkbError, match="error 1:"):
        call()


def test_refusals_leave_the_following_call_unchanged():
    fib, shell, bodies, ops, links, M, Minv, x = make_case(35)
    shell = dict(shell, M=M, Minv=Minv)
    n = bodies["n_nodes"]
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        r0, p0 = fl.apply_system_matvec(x, ETA, dense=dn), fl.apply_system_preconditioner(x, dense=dn)
        args = (bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"])
        _refused(lambda: fl.set_body_operators([n[0], n[1] - 1], *args))                   # node counts
        w = bodies["weights"].copy()
        w[5] = 0.0
        _refused(lambda: fl.set_body_operators(n, w, *args[1:]))                             # a weight <= 0
        bad = links["body"].copy()
        bad[0] = len(n)
        _refused(lambda: fl.set_fiber_links(bad, links["site"], links["rigidity"]))         # body index
        bad[0] = -2
        _refused(lambda: fl.set_fiber_links(bad, links["site"], links["rigidity"]))
        site = links["site"].copy()
        site[0] = bodies["centers"][links["body"][0]]
        _refused(lambda: fl.set_fiber_links(links["body"], site, links["rigidity"]))        # site at the centre
        _refused(lambda: fl.apply_system_matvec(x, ETA, dense=None))                        # dn == NULL, periphery
        _refused(lambda: fl.apply_system_preconditioner(x, dense=None))
        fl.set_target_window(0, fib["pos"].shape[0])  # every fiber row, no periphery or body rows
        fl.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
        _refused(lambda: fl.apply_system_matvec(x, ETA, dense=dn))                          # window
        fl.set_target_window(0, -1)
        fl.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
        fl.set_fiber_preconditioner([np.linalg.inv(A) for A in ops["A"]])
        assert np.array_equal(fl.apply_system_matvec(x, ETA, dense=dn), r0)
        assert np.array_equal(fl.apply_system_preconditioner(x, dense=dn), p0)
        # state that a call drops or never had
        fl.set_body_operators(n, *args)                                                      # no A_inv
        _refused(lambda: fl.apply_system_preconditioner(x, dense=dn))
        fl.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])                   # drops operators, links
        _refused(lambda: fl.apply_system_matvec(x, ETA, dense=dn))
        fl.set_body_operators(n, *args, [np.linalg.inv(A) for A in bodies["A"]])
        _refused(lambda: fl.apply_system_matvec(x, ETA, dense=dn))                          # links dropped
        fl.set_fiber_links(links["body"], links["site"], links["rigidity"])
        assert np.array_equal(fl.apply_system_matvec(x, ETA, dense=dn), r0)
        assert np.array_equal(fl.apply_system_preconditioner(x, dense=dn), p0)
    # a bound fiber whose node count lacks the derivative matrices
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        load(fl, fib, shell, dict(pos=bodies["pos"], normals=bodies["normals"], centers=bodies["centers"]))
        for k in ops["D_1_0"]:
            fl.set_fiber_class(k, ops["D_1_0"][k], ops["P"][k])
        fl.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
        _refused(lambda: fl.set_fiber_links(links["body"], links["site"], links["rigidity"]))
    # a group member
    with skb.Flow(0) as fl:
        load(fl, fib, shell, dict(pos=bodies["pos"], normals=bodies["normals"], centers=bodies["centers"]))
        fl.group_init(0, 2)
        _refused(lambda: fl.set_body_operators(n, *args))
        _refused(lambda: fl.apply_system_matvec(x[:fl.solution_size()], ETA))


def test_system_operator_iterations_match_the_reference_loop():
    import torch
    fib, shell, bodies, ops, links, M, Minv, x0 = make_case(36, n_fibers=24, n_shell=260, n_body_nodes=400)
    shell = dict(shell, M=M, Minv=Minv)
    K = 6
    x = x0.copy()
    for _ in range(K):
        y = sr.system_apply_preconditioner(ops["A"], ops["n_nodes"], Minv, bodies["A"], bodies["n_nodes"], x)
        r, _, _ = sr.system_apply_matvec(fib, shell, bodies, ops, links, M, y, ETA)
        x = r / np.abs(r).max()
    dev = torch.device("cuda", 0)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        op = SystemOperator(fl, dn, ETA, dev)
        got = iterate_system(op, torch.from_numpy(x0).to(dev), K)
        torch.cuda.synchronize()
        got = got.cpu().numpy()
        assert op.launches > 0
    assert rel_max(got, x) < 1e-11, rel_max(got, x)

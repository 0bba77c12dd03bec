"""GPU tests of the whole-vector operator and preconditioner over several devices (include/skelly_b200_flow.h
skb_mflow_apply_system_matvec / _preconditioner): System::apply_matvec (system.cpp:269-324) and ::apply_preconditioner
(:248-262) with the bodies and the fiber-body links, each member computing the links of its own fibers and the members'
partial link forces exchanged through the group window (group_ft_store_kernel / group_ft_reduce_kernel).

Device lists [0], [0, 0], [0, 0, 0] (a device listed twice gives two members on one GPU: the whole exchange protocol
runs), and the real lists when more GPUs are present.  The cases are arranged so that each body's bound fibers fall on
at least two members (every other fiber is bound, the bodies taking turns), the two-member cut of the body rows falls
inside a body, and with three members one member owns no body rows (two bodies of two nodes).  Gate: 1e-12 relative per
block (max-norm and l2), and per body for its node rows and its six rows."""
import numpy as np
import pytest

import body_block_reference as bb
import skellysim_b200 as skb
import system_reference as sr
from conftest import rel_max
from skellysim_b200 import capi
from skellysim_b200.solver_hydro import iterate_system
from test_body_block_ext_cpu import body_case, body_x, k_ft_per_body
from test_gpu_system_matvec import TOL, _check, blocks, make_case, setup_flow

pytestmark = pytest.mark.gpu
ETA = 0.9


def device_lists():
    n = capi.device_count()
    out = [[0], [0, 0], [0, 0, 0]]
    for k in (2, 4, 8):
        if n >= k:
            out.append(list(range(k)))
    return out


def setup_mflow(mf, fib, shell, bodies, ops, links):
    """setup_flow of tests/test_gpu_system_matvec.py on a MultiFlow"""
    mf.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
    mf.set_periphery(shell["pos"], shell["normals"])
    mf.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])
    for n in ops["D_1_0"]:
        mf.set_fiber_class(n, ops["D_1_0"][n], ops["P"][n])
        mf.set_fiber_class_derivatives(n, ops["D_2_0"][n], ops["D_3_0"][n], ops["D_4_0"][n])
    mf.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
    mf.set_fiber_preconditioner([np.linalg.inv(A) for A in ops["A"]])
    mf.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"],
                          [np.linalg.inv(A) for A in bodies["A"]])
    mf.set_fiber_links(links["body"], links["site"], links["rigidity"])
    if shell["pos"].shape[0]:
        mf.set_dense(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, shell["M"])
        mf.set_dense(skb.DENSE_M_INV, shell["Minv"])


def body_slices(bodies):
    off = 0
    for n in bodies["n_nodes"]:
        yield slice(off, off + 3 * n), slice(off + 3 * n, off + 3 * n + 6)
        off += 3 * n + 6


def check_blocks(got, ref, fib, shell, bodies):
    for got_b, ref_b in zip(blocks(got, fib, shell), blocks(ref, fib, shell)):
        _check(got_b, ref_b)
    g_b, r_b = blocks(got, fib, shell)[2], blocks(ref, fib, shell)[2]
    for sl in (s for pair in body_slices(bodies) for s in pair):  # a block-wide max-norm hides a small row
        assert rel_max(g_b[sl], r_b[sl]) <= TOL, (sl, rel_max(g_b[sl], r_b[sl]))


# 40 fibers: below the symmetric kernel's threshold (own rows, plain kernel); 120 x (16..96): symmetric partials and
# pull; 24 fibers with two bodies of two nodes: with three members the last owns no body rows
CASES = {"40": dict(n_fibers=40, nodes=(8, 16, 24, 32), n_body_nodes=600, n_bodies=3),
         "120": dict(n_fibers=120, nodes=(16, 32, 48, 64, 96), n_body_nodes=600, n_bodies=3),
         "tiny_bodies": dict(n_fibers=24, nodes=(8, 16), n_body_nodes=4, n_bodies=2)}


def case(name, seed):
    fib, shell, bodies, ops, links, M, Minv, x = make_case(seed, n_shell=300, **CASES[name])
    return fib, dict(shell, M=M, Minv=Minv), bodies, ops, links, M, Minv, x


@pytest.mark.parametrize("cross", [0, 1])
@pytest.mark.parametrize("name", list(CASES))
def test_system_matvec_matches_the_reference_and_the_single_device(name, cross):
    fib, shell, bodies, ops, links, M, Minv, x = case(name, 51)
    ref, vel, ft = sr.system_apply_matvec(fib, shell, bodies, ops, links, M, x, ETA)
    assert np.count_nonzero(ft) > 0 and np.count_nonzero(vel) > 0  # the links act
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        fl.set_cross(cross)
        single = fl.apply_system_matvec(x, ETA, dense=dn)
    check_blocks(single, ref, fib, shell, bodies)
    for devs in device_lists():
        with skb.MultiFlow(devs) as mf:
            mf.set_cross(cross)
            setup_mflow(mf, fib, shell, bodies, ops, links)
            x0 = x.copy()
            r1 = mf.apply_system_matvec(x, ETA)
            assert mf.stats()["launches"] > 0
            r2 = mf.apply_system_matvec(x, ETA)
            r3 = mf.apply_system_matvec(2.0 * x, ETA)  # the double-buffered window halves alternate
            parts = [mf.partition(g) for g in range(len(devs))]
        assert np.array_equal(x, x0), devs
        assert np.array_equal(r1, r2), f"not reproducible on {devs}"
        check_blocks(r1, ref, fib, shell, bodies)
        check_blocks(r3, 2.0 * ref, fib, shell, bodies)
        for got_b, one_b in zip(blocks(r1, fib, shell), blocks(single, fib, shell)):
            _check(got_b, one_b)
        if len(devs) == 1:
            assert np.array_equal(r1, single)
        if name != "tiny_bodies" and len(devs) == 2:  # the cut of the body rows falls inside body 1
            assert 0 < parts[0][5] - 200 < 200
        if name == "tiny_bodies" and len(devs) == 3:
            assert parts[2][4] == parts[2][5]
        owners = {}  # body -> the members its bound fibers are on
        for f, b in enumerate(links["body"]):
            if b >= 0:
                owners.setdefault(b, set()).update(g for g, p in enumerate(parts) if p[0] <= f < p[1])
        if len(devs) > 1:
            assert all(len(g) >= 2 for g in owners.values()), owners


def test_without_bound_fibers_the_fiber_and_shell_rows_are_the_partial_operator():
    fib, shell, bodies, ops, links, M, Minv, x = case("120", 52)
    nf, ns, nb = fib["pos"].shape[0], shell["pos"].shape[0], bodies["pos"].shape[0]
    x_f, x_s, x_b = blocks(x, fib, shell)
    dens = np.concatenate([x_b[s] for s, _ in body_slices(bodies)]).reshape(nb, 3)
    for devs in device_lists():
        with skb.MultiFlow(devs) as mf:
            setup_mflow(mf, fib, shell, bodies, ops, links)
            mf.set_fiber_links(None)
            res = mf.apply_system_matvec(x, ETA)
            r_f, r_s, v_b = mf.apply_matvec(x_f, x_s.reshape(ns, 3), dens, np.zeros((len(bodies["n_nodes"]), 6)), ETA)
        g_f, g_s, g_b = blocks(res, fib, shell)
        assert np.array_equal(g_f, r_f) and np.array_equal(g_s, r_s.reshape(-1)), devs
        _check(g_b, sr.body_matvec(bodies, v_b, x_b))


def test_links_and_body_sums_entry_by_entry():
    """The zeroed-operator setup of tests/test_gpu_system_ext.py: zero A_ and force_operator_, zero periphery and body
    densities.  The fiber boundary rows are the link rows; with U = omega = 0 the body node rows are the flow of F and L,
    whose rank-order sum of the members' partials adds at most members - 1 roundings; the six rows are zero."""
    from test_gpu_system_ext import N_SHELL
    fib, ops, links, bodies = body_case(81, n_bodies=12, body_nodes=(1, 2, 85, 255, 256, 257, 511))
    rng = np.random.default_rng(82)
    nf, n_b = fib["pos"].shape[0], len(bodies["n_nodes"])
    x_f = rng.normal(size=4 * nf)
    x_b_moving, x_b_still = body_x(rng, bodies, densities=False), body_x(rng, bodies, densities=False, motion=False)
    x_moving = np.concatenate([x_f, np.zeros(3 * N_SHELL), x_b_moving])
    x_still = np.concatenate([x_f, np.zeros(3 * N_SHELL), x_b_still])
    d = rng.normal(size=(N_SHELL, 3))
    d /= np.linalg.norm(d, axis=1)[:, None]
    shell_pos, M = d * np.array([7.8, 4.16, 4.16]), rng.normal(size=(3 * N_SHELL,) * 2)
    le, _, fte = bb.link_terms(fib, ops, links, bodies, x_f, x_b_moving)
    ls, _, fts = bb.link_terms(fib, ops, links, bodies, x_f, x_b_moving, absolute=True)
    first = np.concatenate([[0], np.cumsum(fib["n_nodes"])[:-1]]).astype(int)
    rows = np.array([4 * o + 4 * n - 14 for o, n in zip(first, fib["n_nodes"])])
    t = np.array([0, 1, 2, 4, 5, 6])
    k_ft = k_ft_per_body(links, fib, n_b).max()
    c = bodies["centers"]
    ve = bb.centre_flow(bodies["pos"], c, fte[:, :3], fte[:, 3:], ETA)
    vs = bb.centre_flow(bodies["pos"], c, fts[:, :3], fts[:, 3:], ETA, absolute=True)
    for devs in device_lists()[1:3]:
        with skb.MultiFlow(devs) as mf:
            mf.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
            mf.set_periphery(shell_pos, -d)
            mf.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])
            for n in sorted(ops["D_2_0"]):
                mf.set_fiber_class(n, rng.normal(size=(n, n)), rng.normal(size=(4 * n - 14, 4 * n)))
                mf.set_fiber_class_derivatives(n, ops["D_2_0"][n], ops["D_3_0"][n], rng.normal(size=(n, n)))
            mf.set_fiber_operators([np.zeros((4 * n, 4 * n)) for n in fib["n_nodes"]],
                                   [np.zeros((3 * n, 4 * n)) for n in fib["n_nodes"]], ops["xs"], ops["length_prev"],
                                   [0] * len(fib["n_nodes"]))
            mf.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"])
            mf.set_fiber_links(links["body"], links["site"], links["rigidity"])
            mf.set_dense(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, M)
            res_moving = mf.apply_system_matvec(x_moving, ETA)
            res_still = mf.apply_system_matvec(x_still, ETA)
        r_link = bb.ratio(res_moving[rows[:, None] + t[None, :]], le[:, t], ls[:, t])
        assert r_link.max() <= bb.K_LINK_ROWS, (devs, r_link.max())
        k_v = bb.k_flow(n_b) + k_ft + (len(devs) - 1)
        g_b = blocks(res_still, fib, dict(pos=np.zeros((N_SHELL, 3))))[2]
        node_rows = np.concatenate([g_b[s] for s, _ in body_slices(bodies)])
        r_v = bb.ratio(node_rows, ve.reshape(-1), vs.reshape(-1))
        assert r_v.max() <= k_v, (devs, r_v.max(), k_v)
        x_b = x_b_moving
        assert not np.concatenate([g_b[s6] for _, s6 in body_slices(bodies)]).any()
        res_b = blocks(res_moving, fib, dict(pos=np.zeros((N_SHELL, 3))))[2]
        for (s, s6), n in zip(body_slices(bodies), bodies["n_nodes"]):  # K^T lambda = 0: the six rows are U
            assert np.array_equal(res_b[s6], x_b[s6])
        print(f"\n{devs}: link rows {r_link.max():.2f} (K {bb.K_LINK_ROWS}), body node rows {r_v.max():.2f} "
              f"(K {k_v})")


def test_system_preconditioner():
    fib, shell, bodies, ops, links, M, Minv, x = case("120", 53)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        single = fl.apply_system_preconditioner(x, dense=dn)
    x_f, x_s, x_b = blocks(x, fib, shell)
    ref_s = Minv @ x_s
    for devs in device_lists():
        with skb.MultiFlow(devs) as mf:
            setup_mflow(mf, fib, shell, bodies, ops, links)
            x0 = x.copy()
            y = mf.apply_system_preconditioner(x)
            assert np.array_equal(mf.apply_system_preconditioner(x), y)
        assert np.array_equal(x, x0)
        g_f, g_s, g_b = blocks(y, fib, shell)
        assert np.array_equal(g_f, blocks(single, fib, shell)[0]), devs
        _check(g_s, ref_s)
        for (s, s6), A in zip(body_slices(bodies), bodies["A"]):
            sl = slice(s.start, s6.stop)
            ref_b = np.linalg.inv(A) @ x_b[sl]
            _check(g_b[sl], ref_b)
            r = bb.ratio(g_b[sl], *bb.ext_and_scale(bb.gemv_rows, np.linalg.inv(A), x_b[sl]))
            assert r.max() <= bb.k_gemv(A.shape[0]), (devs, r.max())


@pytest.mark.parametrize("n_members", [2, 3])
def test_isolated_body_preconditioner_inverts_the_matvec(n_members):
    from test_body_block_cpu import bodies_of
    bodies = bodies_of((200,), seed=7)
    A = sr.body_operator(bodies["pos"], bodies["normals"], bodies["centers"][0], bodies["weights"], bodies["ex"],
                         bodies["ey"], bodies["ez"])
    A_inv = np.linalg.inv(A)
    x = np.random.default_rng(8).normal(size=A.shape[0])
    err_np = np.abs(A_inv @ (A @ x) - x).max()
    with skb.MultiFlow([0] * n_members) as mf:
        mf.set_fibers(np.zeros((0, 3)), [], [])
        mf.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
        mf.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])
        mf.set_fiber_operators([], [], np.zeros((0, 3)), [], [])
        mf.set_fiber_preconditioner([])
        mf.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"], [A_inv])
        mf.set_fiber_links(None)
        ax = mf.apply_system_matvec(x, ETA)
        px = mf.apply_system_preconditioner(ax)
    _check(ax, A @ x)
    assert np.abs(px - x).max() <= 32 * err_np, (np.abs(px - x).max(), err_np)


class _MultiFlowOperator:
    """the two operators of skellysim_b200.solver_hydro.iterate_system, through a MultiFlow (host vectors)"""

    def __init__(self, mf, eta, dev):
        import torch
        self.mf, self.eta, self.dev, self.torch = mf, eta, dev, torch
        self.launches = 0

    def _through(self, fn, x):
        y = fn(x.cpu().numpy())
        self.launches += self.mf.stats()["launches"]
        return self.torch.from_numpy(y).to(self.dev)

    def apply(self, x):
        return self._through(lambda v: self.mf.apply_system_matvec(v, self.eta), x)

    def apply_preconditioner(self, x):
        return self._through(self.mf.apply_system_preconditioner, x)


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
    for devs in device_lists()[1:3]:
        with skb.MultiFlow(devs) as mf:
            setup_mflow(mf, fib, shell, bodies, ops, links)
            op = _MultiFlowOperator(mf, ETA, dev)
            got = iterate_system(op, torch.from_numpy(x0).to(dev), K).cpu().numpy()
            assert op.launches > 0
        assert rel_max(got, x) < 1e-11, (devs, rel_max(got, x))


def test_a_new_partition_needs_no_new_body_set_up():
    """set_fibers to another fiber count re-partitions the members and re-runs their group set-up; the whole-vector
    calls lay the members' rows out again themselves, without a new set_body_operators or set_gmres, and give bitwise
    what a MultiFlow set up on the new geometry gives.  Both bodies are cut between members."""
    from test_gpu_system_edges import DT, edge_case, setup_mflow_edges
    kw = dict(n_fibers=40, nodes=(8, 16, 24, 32), n_shell=300, n_body_nodes=600, n_bodies=2)
    old = edge_case(kw, 56)
    # 24 fibers of the same classes, so the classes already set stay valid; the periphery and bodies stay the old ones
    fib, _, _, ops, links, x, params, _, src = edge_case(dict(kw, n_fibers=24), 57)
    shell, bodies = old[1], old[2]

    def calls(mf, x, params, src):
        mf.set_point_sources(*src["points"])
        mf.set_background(*src["background"])
        return [mf.apply_system_matvec(x, ETA), mf.apply_system_preconditioner(x),
                mf.build_system_rhs(*params, DT, ETA, f_external=src["f_ext"], body_forces_torques=src["ft"],
                                    v_growth=src["v_growth"], force_scale=src["force_scale"])]

    with skb.MultiFlow([0, 0, 0]) as mf:
        setup_mflow_edges(mf, *old[:5])
        mf.set_gmres(20)
        calls(mf, old[5], old[6], old[8])
        before = [mf.partition(g) for g in range(3)]
        mf.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
        mf.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
        mf.set_fiber_preconditioner(ops["A_inv"])
        mf.set_fiber_links(links["body"], links["site"], links["rigidity"])
        got = calls(mf, x, params, src)
        parts = [mf.partition(g) for g in range(3)]
    assert parts != before and all(p[4] % 300 and p[4] < p[5] for p in parts[1:]), (before, parts)
    with skb.MultiFlow([0, 0, 0]) as mf:
        setup_mflow_edges(mf, fib, shell, bodies, ops, links)
        want = calls(mf, x, params, src)
        assert [mf.partition(g) for g in range(3)] == parts
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


def _refused(call):
    with pytest.raises(skb.SkbError, match="error [14]:"):  # SKB_ERR_INVALID or SKB_ERR_STATE
        call()


def test_refusals_leave_the_following_call_unchanged():
    fib, shell, bodies, ops, links, M, Minv, x = case("40", 54)
    n = bodies["n_nodes"]
    args = (bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"])
    A_inv = [np.linalg.inv(A) for A in bodies["A"]]
    with skb.MultiFlow([0, 0, 0]) as mf:
        setup_mflow(mf, fib, shell, bodies, ops, links)
        r0, p0 = mf.apply_system_matvec(x, ETA), mf.apply_system_preconditioner(x)

        def unchanged():
            assert np.array_equal(mf.apply_system_matvec(x, ETA), r0)
            assert np.array_equal(mf.apply_system_preconditioner(x), p0)

        _refused(lambda: mf.set_body_operators([n[0], n[1], n[2] - 1], *args, A_inv))     # node counts
        unchanged()
        _refused(lambda: mf.set_body_operators(n[:2], *args, A_inv[:2]))                  # body count
        unchanged()
        w = bodies["weights"].copy()
        w[-5] = 0.0
        _refused(lambda: mf.set_body_operators(n, w, *args[1:], A_inv))                    # a weight <= 0
        unchanged()
        for f_bad, value in ((len(links["body"]) - 2, len(n)), (len(links["body"]) - 2, -2)):  # body index
            bad = links["body"].copy()
            bad[f_bad] = value
            _refused(lambda: mf.set_fiber_links(bad, links["site"], links["rigidity"]))
            unchanged()
        site = links["site"].copy()
        last_bound = int(np.flatnonzero(links["body"] >= 0)[-1])  # a fiber of the last member
        site[last_bound] = bodies["centers"][links["body"][last_bound]]
        _refused(lambda: mf.set_fiber_links(links["body"], site, links["rigidity"]))       # site at the centre
        unchanged()
        # state that a call drops or never had
        mf.set_body_operators(n, *args)                                                      # no A_inv
        _refused(lambda: mf.apply_system_preconditioner(x))
        mf.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])                   # drops operators, links
        _refused(lambda: mf.apply_system_matvec(x, ETA))
        mf.set_body_operators(n, *args, A_inv)
        _refused(lambda: mf.apply_system_matvec(x, ETA))                                    # links dropped
        mf.set_fiber_links(links["body"], links["site"], links["rigidity"])
        unchanged()
        for k in ops["D_1_0"]:                                          # a class drops the links and the operators
            mf.set_fiber_class(k, ops["D_1_0"][k], ops["P"][k])
        _refused(lambda: mf.apply_system_matvec(x, ETA))
        mf.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
        mf.set_fiber_preconditioner([np.linalg.inv(A) for A in ops["A"]])
        _refused(lambda: mf.apply_system_matvec(x, ETA))
        mf.set_fiber_links(links["body"], links["site"], links["rigidity"])
        unchanged()
        mf.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])                          # fibers drop the links
        mf.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
        mf.set_fiber_preconditioner([np.linalg.inv(A) for A in ops["A"]])
        _refused(lambda: mf.apply_system_matvec(x, ETA))
        mf.set_fiber_links(links["body"], links["site"], links["rigidity"])
        unchanged()
        # a periphery of another size: the dense row blocks set for the old one no longer fit and are refused
        nf, ns = fib["pos"].shape[0], shell["pos"].shape[0]
        rng = np.random.default_rng(55)
        d = rng.normal(size=(ns + 30, 3))
        d /= np.linalg.norm(d, axis=1)[:, None]
        mf.set_periphery(d * np.array([7.8, 4.16, 4.16]), -d)
        mf.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
        mf.set_fiber_preconditioner([np.linalg.inv(A) for A in ops["A"]])
        x_new = np.concatenate([x[:4 * nf], rng.normal(size=3 * (ns + 30)), x[4 * nf + 3 * ns:]])
        with pytest.raises(skb.SkbError, match="error 1:.*skb_mflow_set_dense again"):
            mf.apply_system_matvec(x_new, ETA)
        with pytest.raises(skb.SkbError, match="error 1:.*skb_mflow_set_dense again"):
            mf.apply_system_preconditioner(x_new)
        mf.set_periphery(shell["pos"], shell["normals"])  # back to the size the blocks were set for
        mf.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
        mf.set_fiber_preconditioner([np.linalg.inv(A) for A in ops["A"]])
        unchanged()
    # no fiber inverse, no dense operator, a bound fiber whose node count lacks the derivative matrices
    with skb.MultiFlow([0, 0]) as mf:
        mf.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
        mf.set_periphery(shell["pos"], shell["normals"])
        mf.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])
        for k in ops["D_1_0"]:
            mf.set_fiber_class(k, ops["D_1_0"][k], ops["P"][k])
        mf.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
        _refused(lambda: mf.set_fiber_links(links["body"], links["site"], links["rigidity"]))
        mf.set_body_operators(n, *args, A_inv)
        mf.set_fiber_links(None)
        _refused(lambda: mf.apply_system_matvec(x, ETA))                                    # no dense operator
        _refused(lambda: mf.apply_system_preconditioner(x))                                 # no inverse, no M_inv
        mf.set_dense(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, M)
        mf.apply_system_matvec(x, ETA)
        mf.set_fiber_preconditioner([np.linalg.inv(A) for A in ops["A"]])
        _refused(lambda: mf.apply_system_preconditioner(x))                                 # no M_inv
        mf.set_dense(skb.DENSE_M_INV, Minv)
        mf.apply_system_preconditioner(x)
    # the single-device calls keep refusing group members
    with skb.Flow(0) as fl:
        fl.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
        fl.set_periphery(shell["pos"], shell["normals"])
        fl.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])
        fl.group_init(0, 2)
        _refused(lambda: fl.set_body_operators(n, *args))

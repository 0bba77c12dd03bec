"""GPU tests of the whole-vector calls on one rank per GPU (include/skelly_b200_flow.h skb_flow_group_set_body_operators,
_set_fiber_links, _apply_system_matvec_device, _apply_system_preconditioner_device, _build_system_rhs_device): every
member holds only its own rows of the solution vector (distributed.system_rows) and exchanges its body rows -- and for
the preconditioner its periphery rows -- through the group window.

The members live in one process, connected by skb_flow_group_connect, each driven by its own Python thread on its own
stream (ctypes releases the GIL), on device lists [0, 0] and [0, 0, 0] (two or three members on one GPU: the whole
exchange protocol runs) and on the real lists when more GPUs are present.  The cases are those of
tests/test_gpu_mflow_system.py.  Each member's rows, scattered through local_rows, are held bitwise to skb_mflow on the
same device list and at the project's gate (1e-12 relative per block and per body) to tests/system_reference.py and
tests/system_rhs_reference.py.  Every refusal is made on all members at once, so no member ever launches while another
refuses."""
import threading

import numpy as np
import pytest

import skellysim_b200 as skb
import system_reference as sr
from oracle.fiber_fd import compute_matrices
from skellysim_b200 import capi, distributed
from test_gpu_flow import load
from test_gpu_mflow_system import CASES, body_slices, case, check_blocks, setup_mflow
from test_gpu_system_matvec import _check, blocks, setup_flow
from test_gpu_system_rhs import check_rhs, reference

pytestmark = pytest.mark.gpu
ETA, DT = 0.9, 1e-3


def device_lists():
    n = capi.device_count()
    return [[0, 0], [0, 0, 0]] + [list(range(k)) for k in (2, 4) if n >= k]


def rhs_inputs(fib, bodies, ops, seed):
    """the reference's class matrices (the RHS reads them) and the RHS inputs of tests/test_gpu_system_rhs.py"""
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
    return params, fparams, src


def run_all(n, fn):
    """fn(g) on one thread per member at once; the first exception is raised"""
    errs = [None] * n

    def body(g):
        try:
            fn(g)
        except BaseException as e:  # noqa: BLE001 -- handed to the main thread
            errs[g] = e

    th = [threading.Thread(target=body, args=(g,)) for g in range(n)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for e in errs:
        if e is not None:
            raise e


class Members:
    """n connected group members on `devs`, each with its operators, its dense row blocks, its own work vectors and
    stream.  scatter / gather move whole vectors to / from the members' local vectors."""

    def __init__(self, devs, fib, shell, bodies, ops, links, cross=-1, src=None, body_inverse=True):
        import torch
        self.torch, self.n, self.devs = torch, len(devs), devs
        ns, nb = shell["pos"].shape[0], bodies["pos"].shape[0]
        fn = list(fib["n_nodes"])
        off = np.concatenate([[0], np.cumsum(fn)]).astype(int)
        self.parts = [capi.partition_query(fn, ns, nb, self.n, g) for g in range(self.n)]
        self.rows = [distributed.system_rows(p, fn, ns, bodies["n_nodes"]) for p in self.parts]
        self.flows = [skb.Flow(d) for d in devs]
        self.dense = [None] * self.n
        for g, fl in enumerate(self.flows):
            load(fl, fib, shell, dict(pos=bodies["pos"], normals=bodies["normals"], centers=bodies["centers"]))
            fl.set_cross(cross)
            fl.set_target_ranges(*self.parts[g])
            fl.group_init(g, self.n)
        for g, fl in enumerate(self.flows):
            for h, peer in enumerate(self.flows):
                if g != h:
                    fl.group_connect(h, peer)
        for g, fl in enumerate(self.flows):
            fl.group_warmup()
            f0, f1, s0, s1 = self.parts[g][:4]
            for k in ops["D_1_0"]:
                fl.set_fiber_class(k, ops["D_1_0"][k], ops["P"][k])
                if k in ops["D_2_0"]:  # (a class beyond the device build's node counts has none)
                    fl.set_fiber_class_derivatives(k, ops["D_2_0"][k], ops["D_3_0"][k], ops["D_4_0"][k])
            fl.set_fiber_operators(ops["A"][f0:f1], ops["force"][f0:f1], ops["xs"][off[f0]:off[f1]],
                                   ops["length_prev"][f0:f1], ops["plus"][f0:f1])
            fl.set_fiber_preconditioner(ops["A_inv"][f0:f1] if "A_inv" in ops else
                                        [np.linalg.inv(A) for A in ops["A"][f0:f1]])
            fl.group_set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"],
                                        [np.linalg.inv(A) for A in bodies["A"]] if body_inverse else None)
            fl.group_set_fiber_links(links["body"][f0:f1], links["site"][f0:f1], links["rigidity"][f0:f1])
            if s1 > s0:
                self.dense[g] = skb.Dense(device_ids=[devs[g]])
                self.dense[g].set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, shell["M"][3 * s0:3 * s1])
                self.dense[g].set_matrix(skb.DENSE_M_INV, shell["Minv"][3 * s0:3 * s1])
            if src is not None:
                fl.set_point_sources(*src["points"])
                fl.set_background(*src["background"])
        self.size = int(sum(r.size for r in self.rows))
        kw = dict(dtype=torch.float64)
        self.x = [torch.zeros(max(r.size, 1), device=f"cuda:{d}", **kw) for r, d in zip(self.rows, devs)]
        self.y = [torch.zeros(max(r.size, 1), device=f"cuda:{d}", **kw) for r, d in zip(self.rows, devs)]
        self.streams = [torch.cuda.Stream(device=d) for d in devs]
        self.off, self.fib = off, fib

    def close(self):
        for d in self.dense:
            if d is not None:
                d.close()
        for fl in self.flows:
            fl.close()

    def scatter(self, v):
        for g, r in enumerate(self.rows):
            if r.size:
                self.x[g][:r.size].copy_(self.torch.from_numpy(np.ascontiguousarray(v[r])))
        self.torch.cuda.synchronize()

    def gather(self):
        self.torch.cuda.synchronize()
        out = np.full(self.size, np.nan)
        for g, r in enumerate(self.rows):
            out[r] = self.y[g][:r.size].cpu().numpy()
        return out

    def _run(self, call):
        def fn(g):
            st = self.streams[g]
            call(g, self.flows[g], st.cuda_stream)
            st.synchronize()
        run_all(self.n, fn)
        self.torch.cuda.synchronize()

    def matvec(self, v):
        self.scatter(v)
        self._run(lambda g, fl, st: fl.group_apply_system_matvec_device(self.dense[g], self.x[g].data_ptr(), ETA,
                                                                        self.y[g].data_ptr(), st))
        return self.gather()

    def precondition(self, v):
        self.scatter(v)
        self._run(lambda g, fl, st: fl.group_apply_system_preconditioner_device(self.dense[g], self.x[g].data_ptr(),
                                                                                self.y[g].data_ptr(), st))
        return self.gather()

    def rhs(self, params, src):
        torch = self.torch
        ins = []
        for g, d in enumerate(self.devs):
            f0, f1 = self.parts[g][:2]
            fe = torch.from_numpy(np.ascontiguousarray(src["f_ext"][self.off[f0]:self.off[f1]])).to(f"cuda:{d}")
            bf = torch.from_numpy(np.ascontiguousarray(src["ft"][:, :3])).to(f"cuda:{d}")
            bt = torch.from_numpy(np.ascontiguousarray(src["ft"][:, 3:])).to(f"cuda:{d}")
            own = [p[f0:f1] if np.ndim(p) else p for p in params]
            ins.append((fe, bf, bt, own, src["v_growth"][f0:f1], src["force_scale"][f0:f1]))
        torch.cuda.synchronize()
        p = lambda t: t.data_ptr() if t.numel() else 0

        def call(g, fl, st):
            fe, bf, bt, own, vg, fs = ins[g]
            fl.group_build_system_rhs_device(*own, DT, ETA, p(fe), p(bf), p(bt), self.y[g].data_ptr(), v_growth=vg,
                                             force_scale=fs, stream=st)
        self._run(call)
        return self.gather()

    def errors(self):
        return [fl.group_error() for fl in self.flows]


def rhs_case(name, seed):
    fib, shell, bodies, ops, links, M, Minv, x = case(name, seed)
    params, fparams, src = rhs_inputs(fib, bodies, ops, seed)
    return fib, shell, bodies, ops, links, x, params, fparams, src


def mflow_results(devs, fib, shell, bodies, ops, links, x, params, src, cross):
    with skb.MultiFlow(devs) as mf:
        mf.set_cross(cross)
        setup_mflow(mf, fib, shell, bodies, ops, links)
        mf.set_point_sources(*src["points"])
        mf.set_background(*src["background"])
        out = (mf.apply_system_matvec(x, ETA), mf.apply_system_matvec(2.0 * x, ETA), mf.apply_system_preconditioner(x),
               mf.build_system_rhs(*params, DT, ETA, f_external=src["f_ext"], body_forces_torques=src["ft"],
                                   v_growth=src["v_growth"], force_scale=src["force_scale"]))
    return out


@pytest.mark.parametrize("cross", [0, 1])
@pytest.mark.parametrize("name", list(CASES))
def test_members_match_mflow_bitwise_and_the_reference(name, cross):
    fib, shell, bodies, ops, links, x, params, fparams, src = rhs_case(name, 71)
    ref_mv, _, _ = sr.system_apply_matvec(fib, shell, bodies, ops, links, shell["M"], x, ETA)
    ref_pc = sr.system_apply_preconditioner(ops["A"], ops["n_nodes"], shell["Minv"], bodies["A"], bodies["n_nodes"], x)
    ref_rhs = reference(fib, shell, bodies, fparams, src)
    for devs in device_lists():
        m_mv, m_mv2, m_pc, m_rhs = mflow_results(devs, fib, shell, bodies, ops, links, x, params, src, cross)
        mem = Members(devs, fib, shell, bodies, ops, links, cross, src)
        try:
            assert np.array_equal(np.sort(np.concatenate(mem.rows)), np.arange(x.size))  # one owner per row
            mv = mem.matvec(x)
            mv2 = mem.matvec(2.0 * x)  # the other window half
            mv3 = mem.matvec(x)        # back to the first
            pc = mem.precondition(x)
            rhs = mem.rhs(params, src)
            # GMRES's interleaving: P^-1, A, P^-1, A, then the RHS of the next step
            seq = [mem.precondition(x), mem.matvec(x), mem.precondition(2.0 * x), mem.matvec(2.0 * x),
                   mem.rhs(params, src)]
            assert mem.errors() == [-1] * len(devs), devs
        finally:
            mem.close()
        for got, want in ((mv, m_mv), (mv2, m_mv2), (mv3, m_mv), (pc, m_pc), (rhs, m_rhs)):
            assert np.array_equal(got, want), devs
        for got, want in zip(seq, (pc, mv, None, mv2, rhs)):
            if want is not None:
                assert np.array_equal(got, want), devs
        check_blocks(mv, ref_mv, fib, shell, bodies)
        for got_b, ref_b in zip(blocks(pc, fib, shell)[:2], blocks(ref_pc, fib, shell)[:2]):
            _check(got_b, ref_b)
        g_b, r_b = blocks(pc, fib, shell)[2], blocks(ref_pc, fib, shell)[2]
        for nodes, six in body_slices(bodies):  # a body's preconditioned rows, as one block
            _check(g_b[nodes.start:six.stop], r_b[nodes.start:six.stop])
        check_rhs(rhs, ref_rhs, fib, shell, bodies)


def test_a_flow_that_is_no_member_takes_the_single_device_calls():
    import torch
    fib, shell, bodies, ops, links, x, params, fparams, src = rhs_case("40", 72)
    dev = torch.device("cuda", 0)
    n = x.size
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        fl.set_point_sources(*src["points"])
        fl.set_background(*src["background"])
        fl.group_set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"],
                                    [np.linalg.inv(A) for A in bodies["A"]])
        fl.group_set_fiber_links(links["body"], links["site"], links["rigidity"])
        d_x = torch.from_numpy(x).to(dev)
        out = [torch.zeros(n, dtype=torch.float64, device=dev) for _ in range(6)]
        fe = torch.from_numpy(np.ascontiguousarray(src["f_ext"])).to(dev)
        bf = torch.from_numpy(np.ascontiguousarray(src["ft"][:, :3])).to(dev)
        bt = torch.from_numpy(np.ascontiguousarray(src["ft"][:, 3:])).to(dev)
        fl.apply_system_matvec_device(dn, d_x.data_ptr(), ETA, out[0].data_ptr())
        fl.group_apply_system_matvec_device(dn, d_x.data_ptr(), ETA, out[1].data_ptr())
        fl.apply_system_preconditioner_device(dn, d_x.data_ptr(), out[2].data_ptr())
        fl.group_apply_system_preconditioner_device(dn, d_x.data_ptr(), out[3].data_ptr())
        kw = dict(v_growth=src["v_growth"], force_scale=src["force_scale"])
        fl.build_system_rhs_device(*params, DT, ETA, fe.data_ptr(), bf.data_ptr(), bt.data_ptr(), out[4].data_ptr(),
                                   **kw)
        fl.group_build_system_rhs_device(*params, DT, ETA, fe.data_ptr(), bf.data_ptr(), bt.data_ptr(),
                                         out[5].data_ptr(), **kw)
        torch.cuda.synchronize()
    o = [t.cpu().numpy() for t in out]
    for a, b in ((0, 1), (2, 3), (4, 5)):
        assert np.array_equal(o[a], o[b])


def _refused_on_all(mem, call):
    """call(g, fl) on every member; each must refuse before any launch"""
    for g, fl in enumerate(mem.flows):
        with pytest.raises(skb.SkbError, match="error [14]:"):  # SKB_ERR_INVALID or SKB_ERR_STATE
            call(g, fl)


def test_refusals_on_every_member_leave_the_next_call_unchanged():
    fib, shell, bodies, ops, links, x, params, fparams, src = rhs_case("40", 73)
    mem = Members([0, 0, 0], fib, shell, bodies, ops, links, src=src)
    try:
        mv0, pc0 = mem.matvec(x), mem.precondition(x)
        mem.scatter(x)
        p = lambda g: mem.x[g].data_ptr()
        q = lambda g: mem.y[g].data_ptr()
        # no dense block for the own periphery rows
        _refused_on_all(mem, lambda g, fl: fl.group_apply_system_matvec_device(None, p(g), ETA, q(g)))
        _refused_on_all(mem, lambda g, fl: fl.group_apply_system_preconditioner_device(None, p(g), q(g)))
        # a block of one row too few
        wrong = []
        for g, (s0, s1) in enumerate(pp[2:4] for pp in mem.parts):
            d = skb.Dense(device_ids=[0])
            d.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, shell["M"][3 * s0:3 * s1 - 3])
            d.set_matrix(skb.DENSE_M_INV, shell["Minv"][3 * s0:3 * s1 - 3])
            wrong.append(d)
        _refused_on_all(mem, lambda g, fl: fl.group_apply_system_matvec_device(wrong[g], p(g), ETA, q(g)))
        _refused_on_all(mem, lambda g, fl: fl.group_apply_system_preconditioner_device(wrong[g], p(g), q(g)))
        for d in wrong:
            d.close()
        # eta, NULL vectors
        _refused_on_all(mem, lambda g, fl: fl.group_apply_system_matvec_device(mem.dense[g], p(g), 0.0, q(g)))
        _refused_on_all(mem, lambda g, fl: fl.group_apply_system_matvec_device(mem.dense[g], 0, ETA, q(g)))
        _refused_on_all(mem, lambda g, fl: fl.group_apply_system_preconditioner_device(mem.dense[g], p(g), 0))
        # set-up refusals: node counts, body count, a bound fiber's site at its body's centre
        n = bodies["n_nodes"]
        args = (bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"])
        _refused_on_all(mem, lambda g, fl: fl.group_set_body_operators([n[0], n[1], n[2] - 1], *args))
        _refused_on_all(mem, lambda g, fl: fl.group_set_body_operators(n[:2], *args))

        def bad_site(g, fl):
            f0, f1 = mem.parts[g][:2]
            site = links["site"][f0:f1].copy()
            bound = np.flatnonzero(links["body"][f0:f1] >= 0)
            site[bound[0]] = bodies["centers"][links["body"][f0 + bound[0]]]
            fl.group_set_fiber_links(links["body"][f0:f1], site, links["rigidity"][f0:f1])
        _refused_on_all(mem, bad_site)
        assert np.array_equal(mem.matvec(x), mv0)
        assert np.array_equal(mem.precondition(x), pc0)
        # no A_inv: the preconditioner is refused, the matvec is not
        for fl in mem.flows:
            fl.group_set_body_operators(n, *args)
        _refused_on_all(mem, lambda g, fl: fl.group_apply_system_preconditioner_device(mem.dense[g], p(g), q(g)))
        assert np.array_equal(mem.matvec(x), mv0)
        assert mem.errors() == [-1] * 3
    finally:
        mem.close()
    # the fiber rows move between the members while their body rows stay: every buffer was sized for the old split, so
    # all three calls are refused on both members until the set-up runs again
    mem = Members([0, 0], fib, shell, bodies, ops, links, src=src)
    try:
        mem.matvec(x)
        moved = [list(pt) for pt in mem.parts]
        moved[0][1] += 2
        moved[1][0] += 2
        assert moved[0][4:] == list(mem.parts[0][4:]) and moved[1][4:] == list(mem.parts[1][4:])
        for g, fl in enumerate(mem.flows):
            fl.set_target_ranges(*moved[g])
        p = lambda g: mem.x[g].data_ptr()
        q = lambda g: mem.y[g].data_ptr()
        for g, fl in enumerate(mem.flows):
            f0, f1 = moved[g][:2]
            own = [v[f0:f1] if np.ndim(v) else v for v in params]
            with pytest.raises(skb.SkbError, match="error 1:.*every change of the target ranges"):
                fl.group_build_system_rhs_device(*own, DT, ETA, 0, 0, 0, q(g))
        _refused_on_all(mem, lambda g, fl: fl.group_apply_system_matvec_device(mem.dense[g], p(g), ETA, q(g)))
        _refused_on_all(mem, lambda g, fl: fl.group_apply_system_preconditioner_device(mem.dense[g], p(g), q(g)))
        assert mem.errors() == [-1, -1]
    finally:
        mem.close()
    # a group whose body rows were never laid out, and one whose peers are not connected
    with skb.Flow(0) as a, skb.Flow(0) as b:
        for g, fl in enumerate((a, b)):
            load(fl, fib, shell, dict(pos=bodies["pos"], normals=bodies["normals"], centers=bodies["centers"]))
            fl.set_target_ranges(*capi.partition_query(fib["n_nodes"], shell["pos"].shape[0], bodies["pos"].shape[0],
                                                       2, g))
            fl.group_init(g, 2)
        for fl in (a, b):
            with pytest.raises(skb.SkbError, match="error 4:.*not all peers are connected"):
                fl.group_apply_system_matvec_device(None, 0, ETA, 0)
        a.group_connect(1, b)
        b.group_connect(0, a)
        for fl in (a, b):
            with pytest.raises(skb.SkbError, match="error 1:.*skb_flow_group_set_body_operators"):
                fl.group_build_system_rhs_device(1.0, 2.5e-3, 0.0125, 500.0, 1.0, 0, 0, DT, ETA, 0, 0, 0, 0)
    # the single-device calls keep refusing group members
    with skb.Flow(0) as fl:
        load(fl, fib, shell, dict(pos=bodies["pos"], normals=bodies["normals"], centers=bodies["centers"]))
        fl.group_init(0, 2)
        with pytest.raises(skb.SkbError, match="error 1:"):
            fl.set_body_operators(bodies["n_nodes"], *args)


def test_gmres_over_the_members_converges_to_the_single_device_solution():
    """scipy GMRES over a LinearOperator that scatters into the members' local vectors and gathers back, on A P^-1 with
    the members' RHS: straight free fibers in a uniform flow (the setup of tests/test_gpu_system_rhs.py, whose exact
    solution is every fiber advected by dt U).  The single-device solve of the same system is held to
        ||x - x1||_2 <= 4 cond(A) (||r||_2 / ||b||_2 + 64 u) ||x1||_2,   u = 2^-53,
    with r the members' true residual and cond(A) of the assembled system matrix, as the single-device test does."""
    import scipy.sparse.linalg as sla
    import torch
    from skellysim_b200.solver_hydro import SystemOperator
    rng = np.random.default_rng(74)
    n_fibers, n = 6, 16
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
    m = compute_matrices(n)
    dev = torch.device("cuda", 0)
    to = lambda v: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(dev)

    def setup(fl):
        fl.set_fibers(r_fib, [n] * n_fibers, lengths)
        fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_bodies(np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))

    def build(fl, own):
        fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
        fl.build_fiber_operators(*own, DT, ETA)
        fl.group_set_body_operators([], [], np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
        fl.group_set_fiber_links(None)
        fl.set_background([0, 1, 2], np.zeros(3), Uf)

    def solve(A_of, P_of, b, N):
        AP = sla.LinearOperator((N, N), matvec=lambda v: A_of(P_of(v)))
        z, info = sla.gmres(AP, b, rtol=1e-14, atol=0.0, restart=N, maxiter=4)
        return P_of(z)

    with skb.Flow(0) as fl:
        setup(fl)
        build(fl, params)
        op = SystemOperator(fl, None, ETA, dev)
        b1 = op.rhs(params, DT).cpu().numpy()
        N = op.n
        A1 = lambda v: op.apply(to(v)).cpu().numpy()
        x1 = solve(A1, lambda v: op.apply_preconditioner(to(v)).cpu().numpy(), b1, N)
        Afull = np.stack([A1(e) for e in np.eye(N)], axis=1)
    cond = np.linalg.cond(Afull)
    fn = [n] * n_fibers
    flows = [skb.Flow(0) for _ in range(2)]
    try:
        parts = [capi.partition_query(fn, 0, 0, 2, g) for g in range(2)]
        for g, fl in enumerate(flows):
            setup(fl)
            fl.set_target_ranges(*parts[g])
            fl.group_init(g, 2)
        flows[0].group_connect(1, flows[1])
        flows[1].group_connect(0, flows[0])
        ops_ = []
        for g, fl in enumerate(flows):
            fl.group_warmup()
            f0, f1 = parts[g][:2]
            build(fl, tuple(p[f0:f1] if np.ndim(p) else p for p in params))
            ops_.append(distributed.RankSystemOperator(fl, None, None, parts[g], fn, 0, [], ETA, dev))
        streams = [torch.cuda.Stream(device=0) for _ in range(2)]

        def members(method, v):
            out = np.full(N, np.nan)
            xs = [to(v[o.local_rows]) for o in ops_]
            torch.cuda.synchronize()
            res = [None, None]

            def fn_(g):
                with torch.cuda.stream(streams[g]):
                    res[g] = getattr(ops_[g], method)(xs[g])
                streams[g].synchronize()
            run_all(2, fn_)
            for o, r in zip(ops_, res):
                out[o.local_rows] = r.cpu().numpy()
            return out

        res = [None, None]

        def rhs_(g):
            f0, f1 = parts[g][:2]
            with torch.cuda.stream(streams[g]):
                res[g] = ops_[g].rhs(tuple(p[f0:f1] if np.ndim(p) else p for p in params), DT)
            streams[g].synchronize()
        run_all(2, rhs_)
        b = np.full(N, np.nan)
        for o, r in zip(ops_, res):
            b[o.local_rows] = r.cpu().numpy()
        _check(b, b1)
        A = lambda v: members("apply", v)
        xg = solve(A, lambda v: members("apply_preconditioner", v), b, N)
        r = b - A(xg)
        assert [fl.group_error() for fl in flows] == [-1, -1]
    finally:
        for fl in flows:
            fl.close()
    bound = 4 * cond * (np.linalg.norm(r) / np.linalg.norm(b) + 64 * 2.0 ** -53) * np.linalg.norm(x1)
    err = np.linalg.norm(xg - x1)
    print(f"\n|r|/|b| {np.linalg.norm(r) / np.linalg.norm(b):.1e}, cond {cond:.1e}, |x - x1| {err:.1e}, "
          f"bound {bound:.1e}")
    assert err <= bound, (err, bound)


def _rank_main(rank, world, port, case_args, q):
    """one process per GPU: gloo carries connect_group's handles; the member's matvec rows go back through q"""
    import os

    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        fib, shell, bodies, ops, links, x = case_args
        ns, nb = shell["pos"].shape[0], bodies["pos"].shape[0]
        fn = list(fib["n_nodes"])
        part = capi.partition_query(fn, ns, nb, world, rank)
        off = np.concatenate([[0], np.cumsum(fn)]).astype(int)
        f0, f1, s0, s1 = part[:4]
        dev = torch.device("cuda", rank)
        torch.cuda.set_device(dev)
        fl = skb.Flow(rank)
        load(fl, fib, shell, dict(pos=bodies["pos"], normals=bodies["normals"], centers=bodies["centers"]))
        fl.set_target_ranges(*part)
        distributed.connect_group(fl, rank, world)
        for k in ops["D_1_0"]:
            fl.set_fiber_class(k, ops["D_1_0"][k], ops["P"][k])
            fl.set_fiber_class_derivatives(k, ops["D_2_0"][k], ops["D_3_0"][k], ops["D_4_0"][k])
        fl.set_fiber_operators(ops["A"][f0:f1], ops["force"][f0:f1], ops["xs"][off[f0]:off[f1]],
                               ops["length_prev"][f0:f1], ops["plus"][f0:f1])
        fl.set_fiber_preconditioner([np.linalg.inv(A) for A in ops["A"][f0:f1]])
        fl.group_set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"],
                                    [np.linalg.inv(A) for A in bodies["A"]])
        fl.group_set_fiber_links(links["body"][f0:f1], links["site"][f0:f1], links["rigidity"][f0:f1])
        dm = dp = None
        if s1 > s0:
            dm, dp = skb.Dense(device_ids=[rank]), skb.Dense(device_ids=[rank])
            dm.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, shell["M"][3 * s0:3 * s1])
            dp.set_matrix(skb.DENSE_M_INV, shell["Minv"][3 * s0:3 * s1])
        op = distributed.RankSystemOperator(fl, dm, dp, part, fn, ns, bodies["n_nodes"], ETA, dev)
        xl = torch.from_numpy(np.ascontiguousarray(x[op.local_rows])).to(dev)
        dist.barrier()
        mv = op.apply(xl).cpu().numpy().copy()
        pc = op.apply_preconditioner(xl).cpu().numpy().copy()
        torch.cuda.synchronize()
        q.put((rank, op.local_rows, mv, pc, fl.group_error()))
        dist.barrier()
        fl.close()
    finally:
        dist.destroy_process_group()


def test_one_process_per_gpu():
    n = capi.device_count()
    if n < 2:
        pytest.skip("needs two GPUs")
    import socket

    import torch.multiprocessing as mp
    fib, shell, bodies, ops, links, M, Minv, x = case("120", 75)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank_main, args=(r, 2, port, (fib, shell, bodies, ops, links, x), q))
             for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=600) for _ in range(2)]
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    with skb.MultiFlow([0, 1]) as mf:
        setup_mflow(mf, fib, shell, bodies, ops, links)
        m_mv, m_pc = mf.apply_system_matvec(x, ETA), mf.apply_system_preconditioner(x)
    mv, pc = np.full(x.size, np.nan), np.full(x.size, np.nan)
    for rank, rows, a, b, err in got:
        assert err == -1
        mv[rows], pc[rows] = a[:rows.size], b[:rows.size]
    assert np.array_equal(mv, m_mv) and np.array_equal(pc, m_pc)

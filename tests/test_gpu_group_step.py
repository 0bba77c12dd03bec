"""GPU tests of one timestep on one rank per GPU (include/skelly_b200_flow.h skb_flow_group_step_device,
distributed.RankStepper): every member steps its own fibers and reads the others' new positions, errors and body rows
from its own group window, so that all members hold the same geometry and take the same decision.

The members live in one process, connected by skb_flow_group_connect, each driven by its own Python thread on its own
stream, on device lists [0, 0] and [0, 0, 0] and on the real lists when more GPUs are present.  skb_mflow_step runs the
same member step from the library's own threads, on host arrays it slices and uploads itself; each member's info, its
local rows of the solution (scattered through local_rows), its own tensions and the geometry it holds afterwards are
held bitwise to it on the same device list, step after step, so that the Python driver (RankStepper's slices, uploads
and device inputs) is held to the library's.  Each group step runs before the skb_mflow step it is compared with, the
first one straight after set_gmres.  The step must allocate nothing and load no kernel
while a peer on the same device may spin on a flag: every group step here is held to leave the library's buffer
allocation count (skb_buffer_alloc_count) and torch's allocation count unchanged.  A lazy kernel load cannot be seen in
a process where earlier tests already ran the kernels, so one test runs a first group step in a fresh process, before
any step of any kind, and requires that no flag wait timed out (group_error == -1)."""
import contextlib

import numpy as np
import pytest

import skellysim_b200 as skb
import system_reference as sr
from skellysim_b200 import capi, distributed, timestep
from test_gpu_group_system import run_all
from test_gpu_step import ETA, EMPTY, case_params, periphery, set_classes, set_up, step_case, straight_fibers
from test_gpu_system_edges import sphere

pytestmark = pytest.mark.gpu
DT = 0.02
SOLVE = dict(tol=1e-12, num_blocks=200, max_iters=400)


def device_lists():
    n = capi.device_count()
    return [[0, 0], [0, 0, 0]] + [list(range(k)) for k in (2, 3) if n >= k]


def group_case(name, seed=21):
    """FP, FPB (test_gpu_step.step_case); F1B: one fiber bound to the body, so that members own no fiber; F1: one free
    fiber alone, so that members own nothing; BIG: 128 free fibers of 16 nodes (2048 nodes: the symmetric plan) in a
    periphery.  Every case has an external force on its fiber nodes"""
    if name in ("FP", "FPB"):
        case = step_case(name, seed)
    elif name == "F1B":
        case = step_case("FPB", seed)
        case.update(fibers=case["fibers"][:1], lengths=case["lengths"][:1], fiber_body=[0],
                    site_ref=case["site_ref"][:1], clamped=[1])
    elif name == "F1":
        pos, lengths = straight_fibers(1, 16, seed)
        case = dict(fibers=pos, lengths=list(lengths), body=None, n_shell=0, fiber_body=None, site_ref=None,
                    clamped=[0], ft=None)
    else:
        pos, lengths = straight_fibers(128, 16, seed)
        grid = [1.5 * (np.array([f % 8, (f // 8) % 4, f // 32]) - np.array([3.5, 1.5, 1.5])) for f in range(128)]
        pos = [p - np.array([3.0 * f, 0.0, 0.0]) + grid[f] for f, p in enumerate(pos)]
        case = dict(fibers=pos, lengths=list(lengths), body=None, n_shell=60, fiber_body=None, site_ref=None,
                    clamped=[0] * 128, ft=None)
    n_fib = sum(len(p) for p in case["fibers"])
    case["f_ext"] = 0.1 * np.random.default_rng(seed + 1).normal(size=(n_fib, 3))
    return case


class Ranks:
    """the members of one group on `devs`, set up for `case` as test_gpu_step.set_up sets up a flow, each with its
    RankStepper; `step` runs every member's step on its own thread"""

    def __init__(self, devs, case, gmres=True):
        self.n, self.devs, self.case = len(devs), devs, case
        pos = case["fibers"]
        fn = [len(p) for p in pos]
        self.fn = fn
        ns = case["n_shell"]
        b = case["body"]
        nb_nodes = b["n"] if b else 0
        self.parts = [capi.partition_query(fn, ns, nb_nodes, self.n, g) for g in range(self.n)]
        self.flows = [skb.Flow(d) for d in devs]
        self.dense = [None] * self.n
        r_fib = np.concatenate(pos) if pos else EMPTY
        shell = periphery(ns, 5, case.get("nan", False)) if ns else None
        body = None
        if b:
            r, nrm, w = sphere(b["n"], b["R"])
            ex, ey, ez = sr.singularity_vectors(r, nrm, w)
            A = sr.body_operator(r, nrm, np.zeros(3), w, ex, ey, ez)
            body = (r, nrm, w, ex, ey, ez, np.linalg.inv(A))
        for g, fl in enumerate(self.flows):
            fl.set_fibers(r_fib, fn, case["lengths"])
            fl.set_periphery(shell[0], shell[1]) if shell else fl.set_periphery(EMPTY, EMPTY)
            fl.set_bodies(body[0], body[1], np.zeros((1, 3))) if body else fl.set_bodies(EMPTY, EMPTY, EMPTY)
            fl.set_target_ranges(*self.parts[g])
            fl.group_init(g, self.n)
        for g, fl in enumerate(self.flows):
            for h, peer in enumerate(self.flows):
                if g != h:
                    fl.group_connect(h, peer)
        for g, fl in enumerate(self.flows):
            fl.group_warmup()
            if pos:
                set_classes(fl, fn)
            if body:
                fl.group_set_body_frames([b["n"]], body[0], body[1], body[2], body[3], body[4], body[5], [body[6]])
                fl.group_place_bodies(b["c0"][None], b["q0"][None])
            else:
                fl.group_set_body_operators([], [], EMPTY, EMPTY, EMPTY)
            fl.set_background([0, 1, 2], np.zeros(3), np.array([0.3, -0.2, 0.5]))
            s0, s1 = self.parts[g][2:4]
            if s1 > s0:
                self.dense[g] = skb.Dense(device_ids=[devs[g]])
                self.dense[g].set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, shell[2][3 * s0:3 * s1])
                self.dense[g].set_matrix(skb.DENSE_M_INV, shell[3][3 * s0:3 * s1])
        self.steppers = [distributed.RankStepper(fl, self.dense[g], case_params(case), ETA, self.parts[g],
                                                 fiber_body=case["fiber_body"], site_ref=case["site_ref"],
                                                 device=f"cuda:{devs[g]}", **SOLVE)
                         for g, fl in enumerate(self.flows)]
        if gmres:
            for s in self.steppers:
                s.set_gmres(300)  # the workspace of set_up's skb_mflow_set_gmres

    def close(self):
        for d in self.dense:
            if d is not None:
                d.close()
        for fl in self.flows:
            fl.close()

    def on_all(self, fn):
        """fn(g, stepper) on every member's thread at once; the results in rank order"""
        import torch
        out = [None] * self.n

        def body(g):
            torch.cuda.set_device(self.devs[g])
            with torch.cuda.stream(torch.cuda.Stream(device=self.devs[g])):
                out[g] = fn(g, self.steppers[g])
                torch.cuda.current_stream().synchronize()
        run_all(self.n, body)
        return out

    def step(self, dt=DT, **kw):
        """every member's step; held to allocate nothing on the device, neither in the library nor through torch"""
        import torch
        kw = dict(dict(f_external=self.case["f_ext"], body_forces_torques=self.case["ft"]), **kw)
        torch.cuda.synchronize()
        allocs = lambda: [torch.cuda.memory_stats(d).get("allocation.all.allocated", 0) for d in sorted(set(self.devs))]
        before = (capi.buffer_alloc_count(), allocs())
        out = self.on_all(lambda g, s: s.step(dt, **kw))
        assert (capi.buffer_alloc_count(), allocs()) == before, "a group step allocated device memory"
        return out

    def errors(self):
        return [fl.group_error() for fl in self.flows]


@contextlib.contextmanager
def ranks(devs, case, **kw):
    r = Ranks(devs, case, **kw)
    try:
        yield r
    finally:
        r.close()


def mflow_step(mf, case, dt=DT):
    return mf.step(*case_params(case), dt, ETA, f_external=case["f_ext"], body_forces_torques=case["ft"],
                   fiber_body=case["fiber_body"], site_ref=case["site_ref"], **SOLVE)


def check_members(R, infos, x, tension, info, mf):
    """every member's info, local rows, own tensions and geometry against skb_mflow_step's"""
    off = np.concatenate([[0], np.cumsum(R.fn)]).astype(int)
    r_ref = mf.fibers()
    pl_ref = mf.placement() if R.case["body"] else None
    for g, s in enumerate(R.steppers):
        assert infos[g] == info, (g, infos[g], info)
        rows = s.local_rows
        assert np.array_equal(s.x.cpu().numpy(), x[rows]), g
        a, b = off[R.parts[g][0]], off[R.parts[g][1]]
        assert np.array_equal(s.tension.cpu().numpy(), tension[a:b]), g
        assert np.array_equal(s.positions(), r_ref), g
        if pl_ref is not None:
            assert all(np.array_equal(u, v) for u, v in zip(s.placement(), pl_ref)), g
    assert R.errors() == [-1] * R.n


@pytest.mark.parametrize("name", ["FP", "FPB", "F1B", "F1", "BIG"])
def test_members_step_bitwise_as_mflow_over_three_steps(name):
    case = group_case(name)
    for devs in device_lists():
        with skb.MultiFlow(devs) as mf, ranks(devs, case) as R:
            set_up(mf, None, case)
            for k in range(3):
                infos = R.step()
                x, tension, info = mflow_step(mf, case)
                assert np.isfinite(info["fiber_error"]), (devs, k)
                check_members(R, infos, x, tension, info, mf)


def test_a_non_finite_solution_is_installed_by_no_member_and_the_group_stays_in_step():
    """a NaN in the first member's row block of M_inv only: every member refuses the install alike; then a group
    matvec on every member is bitwise skb_mflow_apply_system_matvec"""
    case = dict(group_case("FPB"), nan=True)
    import torch
    for devs in device_lists()[:2]:
        with skb.MultiFlow(devs) as mf, ranks(devs, case) as R:
            set_up(mf, None, case)
            r0, pl0 = mf.fibers(), mf.placement()
            infos = R.on_all(lambda g, s: (setattr(s, "max_iters", 5), s.step(DT))[1])
            for i in infos:
                assert np.isnan(i["fiber_error"]) and i["worst_fiber"] == -1
            same = lambda u, v: u.keys() == v.keys() and np.array_equal([u[k] for k in u], [v[k] for k in u],
                                                                          equal_nan=True)
            assert all(same(i, infos[0]) for i in infos)
            for s in R.steppers:
                assert np.array_equal(s.positions(), r0)
                assert all(np.array_equal(u, v) for u, v in zip(s.placement(), pl0))
            _, _, mi = mf.step(*case_params(case), DT, ETA, fiber_body=case["fiber_body"], site_ref=case["site_ref"],
                               max_iters=5)
            assert np.isnan(mi["fiber_error"])
            x = np.random.default_rng(3).normal(size=mf.solution_size())
            want = mf.apply_system_matvec(x, ETA)
            ys = []

            def mv(g, s):
                xl = torch.from_numpy(np.ascontiguousarray(x[s.local_rows])).to(f"cuda:{devs[g]}")
                y = torch.zeros(max(s.local_rows.size, 1), dtype=torch.float64, device=f"cuda:{devs[g]}")
                s.flow.group_apply_system_matvec_device(s.dense, xl.data_ptr() if s.local_rows.size else 0, ETA,
                                                        y.data_ptr(), torch.cuda.current_stream().cuda_stream)
                torch.cuda.current_stream().synchronize()
                return y[:s.local_rows.size].cpu().numpy()
            ys = R.on_all(mv)
            got = np.full(x.size, np.nan)
            for s, y in zip(R.steppers, ys):
                got[s.local_rows] = y
            assert np.array_equal(got, want)
            assert R.errors() == [-1] * R.n


def test_refusals_on_every_member_change_nothing_and_launch_nothing():
    """each refusal is made by all three members at once (every member owns one fiber, bound or free, and nodes of the
    body); afterwards the step is the step without the refusals"""
    case = group_case("FPB")
    devs = [0, 0, 0]
    with skb.MultiFlow(devs) as mf, ranks(devs, case) as R:
        set_up(mf, None, case)
        assert all(s.nodes[1] > s.nodes[0] for s in R.steppers)
        r0, pl0 = mf.fibers(), mf.placement()
        bad = [dict(dt=0.0), dict(num_blocks=301), dict(ft=np.full((1, 6), np.inf)),
               dict(f_ext=np.full_like(case["f_ext"], np.nan)), dict(fiber_body=np.array([1], dtype=np.int32))]
        for kw in bad:
            def call(g, s, kw=kw):
                saved = (s.num_blocks, s.fiber_body)
                s.num_blocks = kw.get("num_blocks", s.num_blocks)
                s.fiber_body = kw.get("fiber_body", s.fiber_body)
                try:
                    with pytest.raises(skb.SkbError, match="error 1:"):
                        s.step(kw.get("dt", DT), f_external=kw.get("f_ext", case["f_ext"]),
                               body_forces_torques=kw.get("ft", case["ft"]))
                finally:
                    s.num_blocks, s.fiber_body = saved
            before = capi.launch_count()
            R.on_all(call)
            assert capi.launch_count() == before, kw
            for s in R.steppers:
                assert np.array_equal(s.positions(), r0), kw
                assert all(np.array_equal(u, v) for u, v in zip(s.placement(), pl0)), kw
        x, tension, info = mflow_step(mf, case)
        check_members(R, R.step(), x, tension, info, mf)


def test_a_flow_that_is_no_member_steps_as_skb_flow_step():
    import torch
    case = group_case("FPB")
    with contextlib.ExitStack() as stack:
        fl, twin = stack.enter_context(skb.Flow(0)), stack.enter_context(skb.Flow(0))
        dn, dn2 = stack.enter_context(skb.Dense(device_ids=[0])), stack.enter_context(skb.Dense(device_ids=[0]))
        set_up(fl, dn, case)
        set_up(twin, dn2, case)
        kw = dict(dtype=torch.float64, device="cuda:0")
        fe = torch.from_numpy(case["f_ext"]).to("cuda:0")
        F, T = (torch.from_numpy(np.ascontiguousarray(case["ft"][:, k:k + 3])).to("cuda:0") for k in (0, 3))
        x_d = torch.zeros(fl.solution_size(), **kw)
        t_d = torch.zeros(fl.n_fib, **kw)
        for _ in range(2):
            x, t, info = twin.step(*case_params(case), DT, ETA, dense=dn2, f_external=case["f_ext"],
                                   body_forces_torques=case["ft"], fiber_body=case["fiber_body"],
                                   site_ref=case["site_ref"], **SOLVE)
            got = fl.group_step_device(*case_params(case), DT, ETA, dense_matvec=dn, dense_minv=dn,
                                       d_f_external=fe.data_ptr(), d_body_forces=F.data_ptr(),
                                       d_body_torques=T.data_ptr(), fiber_body=case["fiber_body"],
                                       site_ref=case["site_ref"], d_x_local=x_d.data_ptr(), d_tension=t_d.data_ptr(),
                                       **SOLVE)
            torch.cuda.synchronize()
            assert got == info
            assert np.array_equal(x_d.cpu().numpy(), x) and np.array_equal(t_d.cpu().numpy(), t)
            assert np.array_equal(fl.fibers(), twin.fibers())
            assert all(np.array_equal(u, v) for u, v in zip(fl.placement(), twin.placement()))


def test_run_over_rank_steppers_logs_as_run_over_a_multiflow():
    """every member runs timestep.run with the same forces and a collision test that rejects the second step: the
    restore path runs, and every member's log is the MultiFlow Stepper's"""
    case = group_case("FPB")
    forces = lambda t, r: (case["f_ext"], case["ft"])

    def rejecting():
        calls = []

        def collided(r, c):
            calls.append(1)
            return len(calls) == 2
        return collided

    for devs in device_lists()[:2]:
        with skb.MultiFlow(devs) as mf:
            set_up(mf, None, case)
            s = timestep.Stepper(mf, None, case_params(case), ETA, fiber_body=case["fiber_body"],
                                 site_ref=case["site_ref"], **SOLVE)
            want = timestep.run(s, 3 * DT, DT, fiber_error_tol=10.0, forces=forces, collided=rejecting())
            r_want, pl_want = mf.fibers(), mf.placement()
        with ranks(devs, case) as R:
            logs = R.on_all(lambda g, s: timestep.run(s, 3 * DT, DT, fiber_error_tol=10.0, forces=forces,
                                                      collided=rejecting()))
            assert any(not acc for _, _, acc, _ in want[2])
            for got in logs:
                assert got == want
            for s in R.steppers:
                assert np.array_equal(s.positions(), r_want)
                assert all(np.array_equal(u, v) for u, v in zip(s.placement(), pl_want))
            assert R.errors() == [-1] * R.n


def _first_step_main(q):
    """a fresh process: the set-up, then one group step on [0, 0] before any step of any kind"""
    try:
        case = group_case("FPB")
        with ranks([0, 0], case) as R:
            before = capi.buffer_alloc_count()
            infos = R.step()
            q.put((infos, R.errors(), capi.buffer_alloc_count() - before))
    except BaseException as e:  # noqa: BLE001 -- reported to the parent
        q.put(repr(e))


def test_a_first_step_in_a_fresh_process_loads_and_allocates_nothing_inside_the_call():
    """every kernel the step launches is loaded by skb_flow_set_gmres: a lazy load inside the call, while the other
    member on the device spins on a flag, would end in a flag time-out"""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    p = ctx.Process(target=_first_step_main, args=(q,))
    p.start()
    got = q.get(timeout=600)
    p.join(timeout=600)
    assert p.exitcode == 0 and not isinstance(got, str), got
    infos, errors, allocs = got
    assert errors == [-1, -1] and allocs == 0
    assert infos[0] == infos[1] and np.isfinite(infos[0]["fiber_error"])


def _rank_main(rank, world, port, case, q):
    """one process per GPU: gloo carries connect_group's handles; each rank steps twice and sends back its rows"""
    import os

    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.cuda.set_device(rank)
        pos = case["fibers"]
        fn = [len(p) for p in pos]
        b = case["body"]
        part = capi.partition_query(fn, case["n_shell"], b["n"], world, rank)
        fl = skb.Flow(rank)
        fl.set_fibers(np.concatenate(pos), fn, case["lengths"])
        r_s, n_s, M, Minv = periphery(case["n_shell"], 5)
        fl.set_periphery(r_s, n_s)
        r, nrm, w = sphere(b["n"], b["R"])
        ex, ey, ez = sr.singularity_vectors(r, nrm, w)
        A = sr.body_operator(r, nrm, np.zeros(3), w, ex, ey, ez)
        fl.set_bodies(r, nrm, np.zeros((1, 3)))
        fl.set_target_ranges(*part)
        distributed.connect_group(fl, rank, world)
        set_classes(fl, fn)
        fl.group_set_body_frames([b["n"]], r, nrm, w, ex, ey, ez, [np.linalg.inv(A)])
        fl.group_place_bodies(b["c0"][None], b["q0"][None])
        fl.set_background([0, 1, 2], np.zeros(3), np.array([0.3, -0.2, 0.5]))
        dn = None
        s0, s1 = part[2:4]
        if s1 > s0:
            dn = skb.Dense(device_ids=[rank])
            dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, M[3 * s0:3 * s1])
            dn.set_matrix(skb.DENSE_M_INV, Minv[3 * s0:3 * s1])
        s = distributed.RankStepper(fl, dn, case_params(case), ETA, part, fiber_body=case["fiber_body"],
                                    site_ref=case["site_ref"], device=f"cuda:{rank}", **SOLVE)
        s.set_gmres(300)
        dist.barrier()
        out = []
        for _ in range(2):
            info = s.step(DT, f_external=case["f_ext"], body_forces_torques=case["ft"])
            torch.cuda.synchronize()
            out.append((info, s.x.cpu().numpy().copy(), s.positions(), s.placement()))
        q.put((rank, s.local_rows, out, fl.group_error()))
        dist.barrier()
        fl.close()
    finally:
        dist.destroy_process_group()


def test_one_process_per_gpu():
    if capi.device_count() < 2:
        pytest.skip("needs two GPUs")
    import socket

    import torch.multiprocessing as mp
    case = group_case("FPB")
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank_main, args=(r, 2, port, case, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=600) for _ in range(2)]
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    with skb.MultiFlow([0, 1]) as mf:
        set_up(mf, None, case)
        want = [mflow_step(mf, case) + (mf.fibers(), mf.placement()) for _ in range(2)]
    for rank, rows, out, err in got:
        assert err == -1
        for (info, xl, r, pl), (x, _, mi, r_m, pl_m) in zip(out, want):
            assert info == mi and np.array_equal(xl, x[rows]) and np.array_equal(r, r_m)
            assert all(np.array_equal(u, v) for u, v in zip(pl, pl_m))

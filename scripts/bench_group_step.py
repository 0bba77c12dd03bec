"""Times one timestep of the C3 system (3000 fibers x 32 nodes, 6000 periphery nodes, one 400-node body with 200 bound
fibers, as scripts/bench_system_solve.py builds it) with max_iters fixed at 50, so that the solve's convergence does not
set the time, in alternating rounds:
  (a) skb_flow_group_step_device on device list [0, 0]: two group members in one process, each on its own thread and
      stream, connected with skb_flow_group_connect (distributed.RankStepper);
  (b) skb_mflow_step on [0, 0];
  (c) skb_flow_step on device 0.
Each round restores the same starting geometry first.  For (a) it also times the members' solve alone
(skb_flow_group_solve_system_device on the step's own RHS) and reports the step's time outside the solve, and the device
time of group_fiber_step_kernel (torch.profiler, one launch per member and step) with the bytes one launch moves.
Reports the card and its power limit, read in the same run.  --small: a tiny system, plumbing only."""
import argparse
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

import skellysim_b200 as skb  # noqa: E402
from bench_system_solve import card, system  # noqa: E402
from skellysim_b200 import capi, distributed  # noqa: E402


def on_threads(n, fn):
    errs = [None] * n

    def body(g):
        try:
            fn(g)
        except BaseException as e:  # noqa: BLE001 -- re-raised on the main thread
            errs[g] = e
    th = [threading.Thread(target=body, args=(g,)) for g in range(n)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for e in errs:
        if e is not None:
            raise e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-iters", type=int, default=50)
    ap.add_argument("--small", action="store_true")
    a = ap.parse_args()
    import torch
    shape = (40, 32, 200, 100, 10, 4) if a.small else (3000, 32, 6000, 400, 200, 16)
    s = system(*shape)
    n, n_fib = s["n"], s["n_fib"]
    fn = [n] * n_fib
    eta, dt, tol = 1.0, 1e-3, 1e-10
    params = (np.full(n_fib, 1.0), 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)
    body, site = s["links"]
    site_ref = np.where(body[:, None] >= 0, site, 0.0)
    f_ext = np.random.default_rng(1).uniform(-1, 1, (n_fib * n, 3))
    r_b, e, w_b, ex, ey, ez, A_inv = s["body"]
    m = s["mats"]
    q0 = np.array([[1.0, 0.0, 0.0, 0.0]])
    solve = dict(tol=tol, num_blocks=300, max_iters=a.max_iters)
    out = dict(card=card(), shape=dict(fibers=n_fib, nodes=n, periphery=shape[2], body_nodes=shape[3],
                                       bound=shape[4]), max_iters=a.max_iters, devices=[0, 0])

    def geometry(fl, group=False):
        fl.set_fibers(s["r_fib"], fn, [1.0] * n_fib)
        fl.set_periphery(*s["shell"])
        fl.set_bodies(r_b, e, np.zeros((1, 3)))

    def rest(fl, group=False):
        fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
        (fl.group_set_body_frames if group else fl.set_body_frames)([len(w_b)], r_b, e, w_b, ex, ey, ez, [A_inv])
        (fl.group_place_bodies if group else fl.place_bodies)(np.zeros((1, 3)), q0)

    # ---- (c) one flow ----
    fl = skb.Flow(0)
    dn = skb.Dense(device_ids=[0])
    geometry(fl)
    rest(fl)
    dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, s["M"])
    dn.set_matrix(skb.DENSE_M_INV, s["Minv"])
    fl.set_gmres(300)
    # ---- (b) skb_mflow on [0, 0] ----
    mf = skb.MultiFlow([0, 0])
    geometry(mf)
    rest(mf)
    mf.set_dense(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, s["M"])
    mf.set_dense(skb.DENSE_M_INV, s["Minv"])
    mf.set_gmres(300)
    # ---- (a) two group members on [0, 0] ----
    G = 2
    parts = [capi.partition_query(fn, shape[2], shape[3], G, g) for g in range(G)]
    mem = [skb.Flow(0) for _ in range(G)]
    dns = [None] * G
    for g, f in enumerate(mem):
        geometry(f)
        f.set_target_ranges(*parts[g])
        f.group_init(g, G)
    for g, f in enumerate(mem):
        for h in range(G):
            if h != g:
                f.group_connect(h, mem[h])
    for g, f in enumerate(mem):
        f.group_warmup()
        rest(f, group=True)
        s0, s1 = parts[g][2:4]
        if s1 > s0:
            dns[g] = skb.Dense(device_ids=[0])
            dns[g].set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, s["M"][3 * s0:3 * s1])
            dns[g].set_matrix(skb.DENSE_M_INV, s["Minv"][3 * s0:3 * s1])
    steppers = [distributed.RankStepper(f, dns[g], params, eta, parts[g], fiber_body=body, site_ref=site_ref,
                                        device="cuda:0", **solve) for g, f in enumerate(mem)]
    for st in steppers:
        st.set_gmres(300)
    streams = [torch.cuda.Stream(device=0) for _ in range(G)]

    def on_members(fn_g):
        def body_g(g):
            torch.cuda.set_device(0)
            with torch.cuda.stream(streams[g]):
                fn_g(g)
                streams[g].synchronize()
        on_threads(G, body_g)

    def reset_all():
        for f in (fl, mf):
            f.set_fibers(s["r_fib"], fn, [1.0] * n_fib)
            f.place_bodies(np.zeros((1, 3)), q0)
        for f in mem:
            f.set_fibers(s["r_fib"], fn, [1.0] * n_fib)
            f.group_place_bodies(np.zeros((1, 3)), q0)
        torch.cuda.synchronize()

    def group_step():
        on_members(lambda g: steppers[g].step(dt, f_external=f_ext))

    def mflow_step():
        mf.step(*params, dt, eta, f_external=f_ext, fiber_body=body, site_ref=site_ref, **solve)

    def flow_step():
        fl.step(*params, dt, eta, dense=dn, f_external=f_ext, fiber_body=body, site_ref=site_ref, **solve)

    def group_solve():
        """the members' solve alone, on the RHS the step builds (links, build and RHS untimed)"""
        rhs = [torch.zeros(max(st.local_rows.size, 1), dtype=torch.float64, device="cuda:0") for st in steppers]

        def prep(g):
            st = steppers[g]
            f0, f1 = parts[g][:2]
            c, q = mem[g].placement()
            import step_reference as sref
            mem[g].group_set_fiber_links(body[f0:f1], np.array([sref.site(c[0], q[0], site_ref[f])
                                                                for f in range(f0, f1)]).reshape(-1, 3), 2.5e-3)
            mem[g].build_fiber_operators(*st.params, dt, eta)
            a0, b0 = st.nodes
            st._fext[:b0 - a0].copy_(torch.from_numpy(f_ext[a0:b0]))
            mem[g].group_build_system_rhs_device(*st.params, dt, eta, st._fext.data_ptr() if b0 > a0 else 0, 0, 0,
                                                 rhs[g].data_ptr(), stream=streams[g].cuda_stream)
        on_members(prep)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        on_members(lambda g: mem[g].group_solve_system_device(dns[g], dns[g], rhs[g].data_ptr(), eta,
                                                              steppers[g]._x.data_ptr(),
                                                              stream=streams[g].cuda_stream, **solve))
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    def timed(f):
        reset_all()
        t0 = time.perf_counter()
        f()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    timed(group_step), timed(mflow_step), timed(flow_step)  # warm-up
    reset_all()
    group_solve()
    tg, tm, tf, ts = [], [], [], []
    for _ in range(a.reps):
        tg.append(timed(group_step))
        tm.append(timed(mflow_step))
        tf.append(timed(flow_step))
        reset_all()
        ts.append(group_solve())
    med = lambda v: dict(median=float(np.median(v)), min=min(v), max=max(v))
    out["group_step_s"], out["mflow_step_s"], out["flow_step_s"] = med(tg), med(tm), med(tf)
    out["group_solve_s"] = med(ts)
    out["group_step_outside_solve_s"] = float(np.median(tg) - np.median(ts))
    out["group_errors"] = [f.group_error() for f in mem]
    # the fused kernel alone: its device time per launch in a profiled step
    from torch.profiler import ProfilerActivity, profile
    reset_all()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        group_step()
        torch.cuda.synchronize()
    ev = [(e.device_time_total, e.count) for e in prof.key_averages() if "group_fiber_step_kernel" in e.key]
    nodes = max(st.nodes[1] - st.nodes[0] for st in steppers)
    fibers = max(p[1] - p[0] for p in parts)
    stencil = int(np.count_nonzero(m["D_1_0"]))
    # one launch: 4 x 8 B in per own node, D_1_0's stencil, the tension out (8 B per node) and the positions (24 B per
    # node) and errors (8 B per fiber) into each of the G windows
    byt = 32.0 * nodes + 8.0 * stencil + 8.0 * nodes + G * (24.0 * nodes + 8.0 * fibers)
    if ev:
        kt = ev[0][0] / max(ev[0][1], 1) * 1e-6
        out["group_fiber_step_kernel"] = dict(ms=kt * 1e3, launches=ev[0][1], bytes=byt,
                                              share_of_3_35_TBs=byt / kt / 3.35e12)
    else:
        out["group_fiber_step_kernel"] = "not measured (no kernel event in the profile)"
    for d in dns:
        if d is not None:
            d.close()
    for f in mem:
        f.close()
    mf.close()
    dn.close()
    fl.close()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

"""Times one timestep of the C3 system (3000 fibers x 32 nodes, 6000 periphery nodes, one 400-node body with 200 bound
fibers, as scripts/bench_system_solve.py builds it) with max_iters fixed, so that the solve's convergence does not set
the time.  In alternating rounds:
  (a) skb_flow_step, synchronised;
  (b) the composition a caller wrote before it: the existing device calls (links, build, the device RHS and solve), the
      solution's download, the step and fiber error in numpy, set_fibers, place_bodies and set_fiber_links;
  (c) (a) minus the solve alone (skb_flow_solve_system_device on the same system and max_iters);
skb_flow_fiber_error per call, and fiber_step_kernel alone (its device time from torch.profiler in a run of its own)
with its bytes against 3.35 TB/s: the error-only variant skb_flow_fiber_error launches reads 3 x 8 B per node and D_1_0's
stencil and writes 8 B per fiber (the step's variant moves 4 x 8 B in and 4 x 8 B out per node).  Reports the card and its power
limit, read in the same run.  --small: a tiny system, plumbing only."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

import skellysim_b200 as skb  # noqa: E402
import step_reference as st  # noqa: E402
from bench_system_solve import card, system  # noqa: E402


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
    eta, dt, tol = 1.0, 1e-3, 1e-10
    params = (np.full(n_fib, 1.0), 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)
    body, site = s["links"]
    site_ref = np.where(body[:, None] >= 0, site, 0.0)
    f_ext = np.random.default_rng(1).uniform(-1, 1, (n_fib * n, 3))
    r_b, e, w_b, ex, ey, ez, A_inv = s["body"]
    m = s["mats"]
    D = m["D_1_0"]
    q0 = np.array([[1.0, 0.0, 0.0, 0.0]])
    out = dict(card=card(), shape=dict(fibers=n_fib, nodes=n, periphery=shape[2], body_nodes=shape[3],
                                       bound=shape[4]), max_iters=a.max_iters)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        def reset():
            fl.set_fibers(s["r_fib"], [n] * n_fib, [1.0] * n_fib)
            fl.place_bodies(np.zeros((1, 3)), q0)

        fl.set_fibers(s["r_fib"], [n] * n_fib, [1.0] * n_fib)
        fl.set_periphery(*s["shell"])
        fl.set_bodies(r_b, e, np.zeros((1, 3)))
        fl.set_fiber_class(n, D, m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
        fl.set_body_frames([len(w_b)], r_b, e, w_b, ex, ey, ez, [A_inv])
        fl.place_bodies(np.zeros((1, 3)), q0)
        dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, s["M"])
        dn.set_matrix(skb.DENSE_M_INV, s["Minv"])
        fl.set_gmres(300)
        d_b = torch.empty(fl.solution_size(), dtype=torch.float64, device="cuda:0")
        d_x, d_f = torch.empty_like(d_b), torch.empty((n_fib * n, 3), dtype=torch.float64, device="cuda:0")
        kw = dict(dense=dn, f_external=f_ext, fiber_body=body, site_ref=site_ref, tol=tol, max_iters=a.max_iters)

        def step():
            fl.step(*params, dt, eta, **kw)

        def composition():
            c, q = fl.placement()
            fl.set_fiber_links(body, np.array([st.site(c[0], q[0], site_ref[f]) for f in range(n_fib)]), 2.5e-3)
            fl.build_fiber_operators(*params, dt, eta)
            d_f.copy_(torch.from_numpy(f_ext))
            fl.build_system_rhs_device(*params, dt, eta, d_f.data_ptr(), 0, 0, d_b.data_ptr())
            fl.solve_system_device(dn, d_b.data_ptr(), eta, d_x.data_ptr(), tol=tol, max_iters=a.max_iters)
            x = d_x.cpu().numpy()
            nb0 = 4 * n * n_fib + 3 * shape[2] + 3 * shape[3]
            c_new, q_new = st.body_step(c[0], q[0], x[nb0:nb0 + 3], x[nb0 + 3:nb0 + 6], dt)
            sites = [st.site(c_new, q_new, site_ref[f]) for f in range(n_fib)]
            new = [st.repin(p, sites[f]) if body[f] >= 0 else p for f, (p, _) in enumerate(st.fiber_step(x, [n] * n_fib))]
            [st.fiber_error(p, 1.0, D) for p in new]
            fl.set_fibers(np.concatenate(new), [n] * n_fib, [1.0] * n_fib)
            fl.place_bodies(c_new[None], q_new[None])
            fl.set_fiber_links(body, np.array(sites), 2.5e-3)

        def solve_only():
            fl.set_fiber_links(body, site, 2.5e-3)
            fl.build_fiber_operators(*params, dt, eta)
            b = torch.from_numpy(fl.build_system_rhs(*params, dt, eta, f_external=f_ext)).to("cuda:0")
            x = torch.empty_like(b)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fl.solve_system_device(dn, b.data_ptr(), eta, x.data_ptr(), tol=tol, max_iters=a.max_iters)
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        def timed(fn):
            reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        timed(step), timed(composition), solve_only()  # warm-up
        ta, tb, ts = [], [], []
        for _ in range(a.reps):
            ta.append(timed(step))
            tb.append(timed(composition))
            reset()
            ts.append(solve_only())
        med = lambda v: dict(median=float(np.median(v)), min=min(v), max=max(v))
        out["step_s"], out["composition_s"], out["solve_s"] = med(ta), med(tb), med(ts)
        out["step_outside_solve_s"] = float(np.median(ta) - np.median(ts))
        reset()
        k = 200
        fl.fiber_error()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(k):
            fl.fiber_error()
        per = (time.perf_counter() - t0) / k
        stencil = int(np.count_nonzero(D))
        byt = 24.0 * n * n_fib + 8.0 * stencil + 8.0 * n_fib  # the error-only variant: positions in, one error out
        out["fiber_error_call"] = dict(ms=per * 1e3)
        # the kernel alone: its device time in a profiled run of its own
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
            for _ in range(k):
                fl.fiber_error()
            torch.cuda.synchronize()
        us = [e.device_time_total for e in prof.key_averages() if "fiber_step_kernel" in e.key]
        if us:
            kt = us[0] / k * 1e-6
            out["fiber_step_kernel"] = dict(ms=kt * 1e3, bytes=byt, share_of_3_35_TBs=byt / kt / 3.35e12)
        else:
            out["fiber_step_kernel"] = "not measured (no kernel event in the profile)"
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

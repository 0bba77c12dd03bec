"""Times the dynamic instability and the step after it on the C3 system (scripts/bench_system_solve.py: 3 000 x 32 fiber
nodes, 6 000 periphery nodes, one 400-node body) with 3 000 nucleation sites on the body, in alternating rounds:
  (a) skb_flow_dynamic_instability, then skb_flow_step;
  (b) what a caller did before: the model restated in numpy (tests/dynamic_instability_reference.py) on positions
      downloaded from the flow, set_fibers, set_periphery_shape and set_gmres for the new fiber set, then skb_flow_step;
and the three kernels' device time from torch.profiler in a run of its own.  max_iters is fixed so that both arms solve
alike.  Reports the card and its power limit, read in the same run.  --small: a tiny system, plumbing only."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

import dynamic_instability_reference as dr  # noqa: E402
import skellysim_b200 as skb  # noqa: E402
from bench_system_solve import card, system  # noqa: E402
from skellysim_b200 import capi  # noqa: E402

DI = dict(n_nodes=32, v_growth=0.2, f_catastrophe=0.5, v_grow_collision_scale=0.5, f_catastrophe_collision_scale=2.0,
          nucleation_rate=1.0, radius=0.0125, min_length=0.25, bending_rigidity=2.5e-3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-iters", type=int, default=50)
    ap.add_argument("--small", action="store_true")
    a = ap.parse_args()
    import torch
    shape = (40, 32, 200, 100, 0, 4) if a.small else (3000, 32, 6000, 400, 0, 16)
    n_sites = 40 if a.small else 3000
    s = system(*shape)
    n, n_fib = s["n"], s["n_fib"]
    eta, dt, tol = 1.0, 1e-2, 1e-10
    r_b, e, w_b, ex, ey, ez, A_inv = s["body"]
    i = np.arange(n_sites)
    z = 1.0 - (2 * i + 1) / n_sites
    th = np.pi * (3.0 - np.sqrt(5.0)) * i
    site_ref = 0.5 * np.stack([np.sqrt(1 - z * z) * np.cos(th), np.sqrt(1 - z * z) * np.sin(th), z], axis=1)
    m = s["mats"]
    c0, q0 = np.zeros((1, 3)), np.array([[1.0, 0.0, 0.0, 0.0]])
    p0 = capi.fiber_params(n_fib, 1.0, 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)
    binding0 = np.full((n_fib, 2), -1, dtype=np.int32)
    pinned0 = np.zeros(n_fib, dtype=np.int32)
    sphere = dict(kind=capi.PERIPHERY_SPHERE, a=12.0)
    out = dict(card=card(), shape=dict(fibers=n_fib, nodes=n, periphery=shape[2], body_nodes=shape[3], sites=n_sites),
               dynamic_instability=DI, dt=dt, max_iters=a.max_iters)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        def reset():
            fl.set_fibers(s["r_fib"], [n] * n_fib, [1.0] * n_fib)
            fl.set_periphery_shape(**sphere)
            fl.set_gmres(300)
            fl.place_bodies(c0, q0)

        fl.set_fibers(s["r_fib"], [n] * n_fib, [1.0] * n_fib)
        fl.set_periphery(*s["shell"])
        fl.set_bodies(r_b, e, c0)
        fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
        fl.set_body_frames([len(w_b)], r_b, e, w_b, ex, ey, ez, [A_inv])
        fl.place_bodies(c0, q0)
        fl.set_nucleation_sites([n_sites], site_ref)
        dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, s["M"])
        dn.set_matrix(skb.DENSE_M_INV, s["Minv"])
        reset()

        def step(res):
            body = res["binding"][:, 0]
            sr = site_ref[np.where(body >= 0, res["binding"][:, 1], 0)]
            pr = res["params"]
            fl.step(*(pr[k] for k in capi.FIBER_PARAMS_DTYPE.names), dt, eta, dense=dn, fiber_body=body, site_ref=sr,
                    v_growth=res["v_growth"], tol=tol, max_iters=a.max_iters)

        def device(call):
            res = fl.dynamic_instability(DI, dt, 1, call, p0, binding0, pinned0)
            step(res)
            return res["removed"], res["nucleated"]

        def host(call):
            c, q = fl.placement()
            res = dr.dynamic_instability(DI, dt, 1, call, np.ones(n_fib), p0, binding0, pinned0, [n_sites], site_ref,
                                         c, q, n_nodes_in=[n] * n_fib, r_fib=fl.fibers())
            res["lengths"] = np.asarray(res["lengths"])
            fl.set_fibers(res["positions"], res["n_nodes"], res["lengths"])
            fl.set_periphery_shape(**sphere)
            fl.set_gmres(300)
            step(res)
            return res["removed"], res["nucleated"]

        def timed(fn, call):
            reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            counts = fn(call)
            torch.cuda.synchronize()
            return time.perf_counter() - t0, counts

        timed(device, 0), timed(host, 0)  # warm-up
        ta, tb = [], []
        for r in range(a.reps):
            t, ca = timed(device, r + 1)
            ta.append(t)
            t, cb = timed(host, r + 1)
            tb.append(t)
            assert ca == cb, (ca, cb)  # the same model: the same removals and nucleations
        med = lambda v: dict(median=float(np.median(v)), min=min(v), max=max(v))
        out["device_di_and_step_s"], out["host_di_and_step_s"] = med(ta), med(tb)
        out["removed_nucleated_last"] = list(ca)
        from torch.profiler import ProfilerActivity, profile
        k = 20
        reset()
        fl.dynamic_instability(DI, dt, 1, 0, p0, binding0, pinned0)
        with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
            for c in range(k):
                reset()
                fl.dynamic_instability(DI, dt, 1, c, p0, binding0, pinned0)
            torch.cuda.synchronize()
        for name in ("di_decide_kernel", "di_scan_kernel", "di_compact_kernel"):
            ev = [e for e in prof.key_averages() if name in e.key]
            out[name + "_us"] = (ev[0].device_time_total / ev[0].count) if ev else "not measured (no kernel event)"
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

"""Times one timestep of the C3 system (scripts/bench_system_step.py) inside the reference's ellipsoid (a, b, c = 7.8,
4.16, 4.16; f_0 = 20, l_0 = 0.05) with max_iters fixed, in alternating rounds:
  (a) skb_flow_step with the periphery's shape set (the repulsion and the collision test on the device);
  (b) what a caller did before: the positions from the flow, the repulsion and the collision test in numpy
      (tests/periphery_reference.py), then skb_flow_step with the repulsion as f_external;
and periphery_kernel alone (its device time from torch.profiler in a run of its own) with its bytes against 3.35 TB/s:
the force pass reads 24 B and writes 24 B per node.  Reports the card and its power limit, read in the same run.
--small: a tiny system, plumbing only."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

import periphery_reference as pr  # noqa: E402
import skellysim_b200 as skb  # noqa: E402
from bench_system_solve import card, system  # noqa: E402
from skellysim_b200 import capi  # noqa: E402

SHAPE = dict(kind="ellipsoid", a=7.8, b=4.16, c=4.16, f_0=20.0, l_0=0.05, binding_active=0, polar_angle_start=0.0,
             polar_angle_end=np.pi, binding_threshold=0.75)


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
    q0 = np.array([[1.0, 0.0, 0.0, 0.0]])
    out = dict(card=card(), shape=dict(fibers=n_fib, nodes=n, periphery=shape[2], body_nodes=shape[3],
                                       bound=shape[4]), ellipsoid=[SHAPE["a"], SHAPE["b"], SHAPE["c"]],
               max_iters=a.max_iters)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        def reset():
            fl.set_fibers(s["r_fib"], [n] * n_fib, [1.0] * n_fib)
            fl.place_bodies(np.zeros((1, 3)), q0)

        fl.set_fibers(s["r_fib"], [n] * n_fib, [1.0] * n_fib)
        fl.set_periphery(*s["shell"])
        fl.set_bodies(r_b, e, np.zeros((1, 3)))
        fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
        fl.set_body_frames([len(w_b)], r_b, e, w_b, ex, ey, ez, [A_inv])
        fl.place_bodies(np.zeros((1, 3)), q0)
        dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, s["M"])
        dn.set_matrix(skb.DENSE_M_INV, s["Minv"])
        fl.set_gmres(300)
        kw = dict(dense=dn, fiber_body=body, site_ref=site_ref, tol=tol, max_iters=a.max_iters)
        on = lambda: fl.set_periphery_shape(capi.PERIPHERY_ELLIPSOID, SHAPE["a"], SHAPE["b"], SHAPE["c"],
                                            SHAPE["f_0"], SHAPE["l_0"], SHAPE["binding_active"])
        off = lambda: fl.set_periphery_shape(capi.PERIPHERY_NONE, 0.0)
        is_clamped = np.asarray(body) >= 0

        def device_step():
            fl.step(*params, dt, eta, f_external=f_ext, **kw)

        def host_step():
            r = fl.fibers()
            f = pr.fiber_interaction(SHAPE, r)  # minus_clamped_ = 0 for every fiber here
            fl.step(*params, dt, eta, f_external=f_ext + f, **kw)
            out_ = pr.outside(SHAPE, fl.fibers()).reshape(n_fib, n)
            out_[is_clamped, 0] = False
            return bool(out_.any())

        def timed(fn, shaped):
            reset()
            on() if shaped else off()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        timed(device_step, True), timed(host_step, False)  # warm-up
        ta, tb = [], []
        for _ in range(a.reps):
            ta.append(timed(device_step, True))
            tb.append(timed(host_step, False))
        med = lambda v: dict(median=float(np.median(v)), min=min(v), max=max(v))
        out["device_shape_step_s"], out["host_repulsion_step_s"] = med(ta), med(tb)
        reset()
        on()
        k = 200
        fl.periphery_interaction()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
            for _ in range(k):
                fl.periphery_interaction()
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "periphery_kernel" in e.key and "add" not in e.key]
        byt = 48.0 * n * n_fib
        if ev:
            # each call launches the force pass and the collision pass (which writes no force): the mean of both
            kt = ev[0].device_time_total / ev[0].count * 1e-6
            out["periphery_kernel"] = dict(ms_per_launch=kt * 1e3, launches=ev[0].count, bytes_force_pass=byt,
                                           share_of_3_35_TBs=byt / kt / 3.35e12)
        else:
            out["periphery_kernel"] = "not measured (no kernel event in the profile)"
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

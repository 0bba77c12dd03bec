"""Times the listener's frame of a step on the C3 system (3000 fibers x 32 nodes, 6000 periphery nodes, one 400-node
body with 200 bound fibers, as scripts/bench_system_step.py builds it), from a solution vector and tension on the device.
In alternating rounds, medians of --reps:
  (a) skb_flow_set_listener_state_device: host wall time, and its elapsed stream time (skb_flow_last_stats device_ms,
      which spans the whole call: the host waits between its stages are in it);
  (b) skb_flow_set_listener_state (host x and tension): host wall time;
  (c) the composition a caller needs without it: the solution's download, skb_flow_build_fiber_operators, the packing of
      [x; y; z; T] on the host, skb_flow_apply_fiber_force, the link conditions on the host (tests/system_reference.py,
      xs_ from D_1_0 on the host) and skb_flow_set_listener_frame.
Then, in a torch.profiler run of its own, the device time of the state call's kernels and copies, per kernel: what
the call costs the GPU.  Reports the card and its power limit, read in the same run.  --small: a tiny system, plumbing only."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

import skellysim_b200 as skb  # noqa: E402
import system_reference as sr  # noqa: E402
from bench_system_solve import card, system  # noqa: E402
from skellysim_b200 import capi  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--small", action="store_true")
    a = ap.parse_args()
    import torch
    shape = (40, 32, 200, 100, 10, 4) if a.small else (3000, 32, 6000, 400, 200, 16)
    s = system(*shape)
    n, n_fib, ns, nbn = s["n"], s["n_fib"], shape[2], shape[3]
    eta, dt = 1.0, 1e-3
    params = (np.full(n_fib, 1.0), 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)
    body, site = s["links"]
    r_b, e, w_b, ex, ey, ez, A_inv = s["body"]
    m = s["mats"]
    kind, radii = np.array([1], dtype=np.int32), np.array([[0.5, 0.5, 0.5]])
    out = dict(card=card(), shape=dict(fibers=n_fib, nodes=n, periphery=ns, body_nodes=nbn, bound=shape[4]),
               reps=a.reps)
    with skb.Flow(0) as fl:
        fl.set_fibers(s["r_fib"], [n] * n_fib, [1.0] * n_fib)
        fl.set_periphery(*s["shell"])
        fl.set_bodies(r_b, e, np.zeros((1, 3)))
        fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
        fl.set_body_frames([nbn], r_b, e, w_b, ex, ey, ez, [A_inv])
        fl.place_bodies(np.zeros((1, 3)), np.array([[1.0, 0.0, 0.0, 0.0]]))
        fl.set_fiber_links(body, site, 2.5e-3)
        rng = np.random.default_rng(2)
        x_h, t_h = rng.uniform(-1, 1, fl.solution_size()), rng.uniform(-1, 1, n_fib * n)
        d_x, d_t = torch.from_numpy(x_h).cuda(), torch.from_numpy(t_h).cuda()
        nf = n_fib * n
        xs_of = (2.0 / 1.0) * np.einsum("ji,fjk->fik", m["D_1_0"], s["r_fib"].reshape(n_fib, n, 3)).reshape(-1, 3)
        bodies = dict(n_nodes=[nbn], centers=np.zeros((1, 3)))
        links = dict(body=body, site=site, rigidity=np.full(n_fib, 2.5e-3))
        fib = dict(n_nodes=[n] * n_fib, lengths=[1.0] * n_fib)

        def state_device():
            capi.set_listener_state_device(fl, *params, dt, eta, d_t.data_ptr(), d_x.data_ptr(), kind, radii)
            return fl.stats()["device_ms"]

        def state_host():
            capi.set_listener_state(fl, *params, dt, eta, t_h, x_h, kind, radii)

        def composition():
            x = d_x.cpu().numpy()
            t = d_t.cpu().numpy()
            fl.build_fiber_operators(*params, dt, eta)
            r = fl.fibers().reshape(n_fib, n, 3)
            packed = np.concatenate([r.transpose(0, 2, 1).reshape(n_fib, 3 * n), t.reshape(n_fib, n)], axis=1)
            ff = fl.apply_fiber_force(packed.reshape(-1))
            ops = dict(xs=xs_of, length_prev=[1.0] * n_fib, D_2_0={n: m["D_2_0"]}, D_3_0={n: m["D_3_0"]})
            xb = x[4 * nf + 3 * ns:]
            _, ft = sr.link_conditions(fib, ops, links, bodies, packed.reshape(-1), xb)
            fl.set_listener_frame(ff, x[4 * nf:4 * nf + 3 * ns].reshape(-1, 3), xb[:3 * nbn].reshape(-1, 3), ft,
                                  xb[3 * nbn:3 * nbn + 6][None], kind, radii, eta)

        def timed(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn()
            torch.cuda.synchronize()
            return time.perf_counter() - t0, r

        timed(state_device), timed(state_host), timed(composition)  # warm-up
        ta, tdev, tb, tc = [], [], [], []
        for _ in range(a.reps):
            w, d = timed(state_device)
            ta.append(w)
            tdev.append(d * 1e-3)
            tb.append(timed(state_host)[0])
            tc.append(timed(composition)[0])
        med = lambda v: dict(median=float(np.median(v)), min=float(min(v)), max=float(max(v)))  # noqa: E731
        out["state_device_s"], out["state_device_stream_elapsed_s"] = med(ta), med(tdev)
        out["state_host_s"], out["composition_s"] = med(tb), med(tc)
        out["composition_over_state_device"] = float(np.median(tc) / np.median(ta))
        # the kernels and copies of the call alone (device time per call, from a profiled run of its own)
        from torch.profiler import ProfilerActivity, profile
        k = 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(k):
                state_device()
            torch.cuda.synchronize()
        per = {e.key: e.device_time_total / k * 1e-3 for e in prof.key_averages()
               if e.device_time_total > 0 and ("_kernel" in e.key or e.key.startswith("Memcpy"))}
        if per:
            out["state_device_kernels_ms"] = dict(total=sum(per.values()),
                                                  per_kernel=dict(sorted(per.items(), key=lambda kv: -kv[1])))
        else:
            out["state_device_kernels_ms"] = "not measured (no kernel event in the profile)"
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

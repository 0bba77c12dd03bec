"""Times skb_flow_listener_gradient on the C3 frame (3000 fibers x 32 nodes, 6000 periphery nodes, one 400-node body,
the geometry of scripts/bench_listener_state.py with random strengths) at a 64^3 grid of targets inside the periphery.
In alternating rounds, medians (min-max) of --reps host wall times around a device synchronise:
  (1) capi.listener_gradient;  (2) velocity_field at the same targets;  (3) the gradient by central differences, six
  velocity_field calls.
Then, in a torch.profiler run of its own, the device time per call of every kernel of (1), and the pair rate of the
two gradient pair kernels (the pair_sum_kernel instantiations of kinds 2 and 3).  Reports the card and its power limit,
read in the same run.  --small: a tiny system and grid, plumbing only."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "scripts")]

import skellysim_b200 as skb  # noqa: E402
from bench_system_solve import card, system  # noqa: E402
from skellysim_b200 import capi  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--small", action="store_true")
    a = ap.parse_args()
    import torch
    shape = (40, 32, 200, 100, 10, 4) if a.small else (3000, 32, 6000, 400, 200, 16)
    side = 8 if a.small else 64
    s = system(*shape)
    n, n_fib, ns, nbn = s["n"], s["n_fib"], shape[2], shape[3]
    eta = 1.0
    r_b, e = s["body"][0], s["body"][1]
    g = np.linspace(-3.0, 3.0, side)
    r = np.stack(np.meshgrid(g, 0.5 * g, 0.5 * g, indexing="ij"), axis=-1).reshape(-1, 3)
    rng = np.random.default_rng(3)
    out = dict(card=card(), shape=dict(fibers=n_fib, nodes=n, periphery=ns, body_nodes=nbn, targets=len(r)),
               reps=a.reps)
    with skb.Flow(0) as fl:
        fl.set_fibers(s["r_fib"], [n] * n_fib, [1.0] * n_fib)
        fl.set_periphery(*s["shell"])
        fl.set_bodies(r_b, e, np.zeros((1, 3)))
        fl.set_listener_frame(rng.uniform(-1, 1, (n * n_fib, 3)), rng.uniform(-1, 1, (ns, 3)),
                              rng.uniform(-1, 1, (nbn, 3)), rng.uniform(-1, 1, (1, 6)), rng.uniform(-1, 1, (1, 6)),
                              np.array([1], dtype=np.int32), np.array([[0.5, 0.5, 0.5]]), eta)
        h = 1e-6

        def fd():
            G = np.empty((len(r), 3, 3))
            for j in range(3):
                dx = np.zeros(3)
                dx[j] = h
                G[:, :, j] = (fl.velocity_field(r + dx) - fl.velocity_field(r - dx)) / (2 * h)
            return G

        calls = dict(gradient=lambda: capi.listener_gradient(fl, r), velocity=lambda: fl.velocity_field(r),
                     central_differences=fd)

        def timed(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        for fn in calls.values():
            timed(fn)
        t = {k: [] for k in calls}
        for _ in range(a.reps):
            for k, fn in calls.items():
                t[k].append(timed(fn))
        med = lambda v: dict(median=float(np.median(v)), min=float(min(v)), max=float(max(v)))  # noqa: E731
        out["seconds"] = {k: med(v) for k, v in t.items()}
        out["central_differences_over_gradient"] = float(np.median(t["central_differences"]) /
                                                         np.median(t["gradient"]))
        from torch.profiler import ProfilerActivity, profile
        k = 3
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(k):
                calls["gradient"]()
            torch.cuda.synchronize()
        per = {ev.key: ev.device_time_total / k * 1e-3 for ev in prof.key_averages() if ev.device_time_total > 0}
        out["gradient_kernels_ms"] = dict(sorted(per.items(), key=lambda kv: -kv[1]))
        pair_ms = {kind: sum(v for key, v in per.items() if f"pair_sum_kernel<{kind}," in key) for kind in (2, 3)}
        pairs = {2: (n * n_fib + 1) * len(r), 3: (ns + nbn) * len(r)}
        out["gradient_pair_kernels"] = {
            ("stokeslet" if kind == 2 else "stresslet"): dict(
                ms=pair_ms[kind], pairs=pairs[kind],
                gpairs_per_s=(pairs[kind] / (pair_ms[kind] * 1e-3) * 1e-9) if pair_ms[kind] > 0 else "not measured")
            for kind in (2, 3)}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

"""Cost of placing a rigid body on the device (skb_flow_place_bodies, include/skelly_b200_flow.h) against the host path
it replaces, for one sphere body of 400 and of 2000 nodes (Fibonacci nodes, equal quadrature weights).  In alternating
rounds, one of each per round:
  (a) skb_flow_place_bodies at a random orientation                 host wall time, ending in a synchronise
  (b) the host path: float64 singularity_vectors, body_operator, the inverse (numpy), and skb_flow_set_bodies +
      skb_flow_set_body_operators uploading them                    host wall time of each part
Then, in a profiled pass of its own, the device time of body_place_kernel (torch.profiler, CUDA activities) and its
effective bandwidth: the body-frame inverse and E read once, the placed ones written once, over the kernel time,
against the 3.35 TB/s of the H100 SXM data sheet.  Reports medians and min / max spreads; the card's name and power
limit are read by the same run.  Needs a GPU; there is no CPU path.

    python scripts/bench_body_placement.py [--reps 5] [--json out.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import skellysim_b200 as skb  # noqa: E402
import body_placement_reference as bp  # noqa: E402
import system_reference as sr  # noqa: E402
from bench_system_rhs import card  # noqa: E402

HBM_TBS = 3.35


def run(torch, n, reps):
    rng = np.random.default_rng(n)
    r0, n0, w = bp.sphere_body(n)
    E0 = sr.singularity_vectors(r0, n0, w)
    A0 = sr.body_operator(r0, n0, np.zeros(3), w, *E0)
    c = np.zeros((1, 3))
    spread = lambda a: [float(np.min(a)), float(np.max(a))]
    with skb.Flow(0) as fl:
        fl.set_fibers(np.zeros((0, 3)), [], [])
        fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_bodies(r0, n0, c)
        fl.set_fiber_operators([], [], np.zeros((0, 3)), [], [])
        fl.set_body_frames([n], r0, n0, w, *E0, [np.linalg.inv(A0)])

        def place():
            q = bp.random_quaternions(rng, 1)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fl.place_bodies(c, q)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3

        def host_path():
            q = bp.random_quaternions(rng, 1)
            t = [time.perf_counter()]
            pos, nrm = bp.placed_geometry(r0, n0, c[0], q[0])
            E = sr.singularity_vectors(pos, nrm, w)
            t.append(time.perf_counter())
            A = sr.body_operator(pos, nrm, c[0], w, *E)
            t.append(time.perf_counter())
            Ai = np.linalg.inv(A)
            t.append(time.perf_counter())
            fl.set_bodies(pos, nrm, c)
            fl.set_body_operators([n], w, *E, [Ai])
            torch.cuda.synchronize()
            t.append(time.perf_counter())
            return np.diff(t) * 1e3

        place()  # warm-up
        tp, th = [], []
        for _ in range(reps):
            tp.append(place())
            th.append(host_path())
        th = np.array(th)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                place()
        kern = [e.time_range.elapsed_us() for e in prof.events() if "body_place_kernel" in e.name]
    m = 3 * n + 6
    bytes_moved = 2 * 8 * m * m + 2 * 72 * n
    k_ms = float(np.median(kern)) / 1e3 if kern else float("nan")
    names = ("singularity_vectors", "body_operator", "inverse", "set_bodies_and_upload")
    return dict(nodes=n, place_wall_ms=float(np.median(tp)), place_wall_ms_spread=spread(tp),
                place_kernel_ms=k_ms, place_kernel_ms_spread=spread(np.array(kern) / 1e3) if kern else None,
                bytes_moved=bytes_moved, effective_TBs=bytes_moved / (k_ms * 1e-3) / 1e12,
                share_of_hbm_datasheet=bytes_moved / (k_ms * 1e-3) / 1e12 / HBM_TBS,
                host_path_ms={k: float(np.median(th[:, i])) for i, k in enumerate(names)},
                host_path_total_ms=float(np.median(th.sum(axis=1))),
                host_path_total_ms_spread=spread(th.sum(axis=1)), reps=int(reps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_body_placement.py needs a GPU")
    out = dict(card=card(), bodies=[run(torch, n, a.reps) for n in (400, 2000)])
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

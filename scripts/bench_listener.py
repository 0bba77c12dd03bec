"""Cost of the listener's streamlines and vortex lines on the device (skb_flow_listener_lines,
include/skelly_b200_flow.h) against the reference's one-line-at-a-time pattern.

The geometry is the C3 system of scripts/bench_system_solve.py (3000 fibers x 32 nodes, 6000 periphery nodes on a
sphere of radius 6, one 400-node sphere of radius 0.5), with the same seed.  The strengths are seeded random strengths
of that system's size: the library's solve returns the solution vector, and turning it into the frame's strengths is
the caller's part.  The reader's defaults (dt_init 0.1, t_final 1, abs_err 1e-10, rel_err 1e-6, back and forward).
In alternating rounds, host wall time around synchronised calls:
  (a) 1024 streamlines seeded inside the periphery, one call
  (b) 256 vortex lines, one call
  (c) the first 16 of (a)'s seeds the reference's way: tests/streamline_reference.py on the host, calling
      skb_flow_velocity_at_targets (its graphed 1-6 target path) once per stage
Reports the card's name and power limit (read by the same run), per-line times, the 16 lines' agreement between (a)
and (c), and in a run of its own a torch.profiler split of (a): pair-sum kernels, the listener's kernels, the rest,
and the gaps.  Needs a GPU; --small runs everything at a tiny size.

    python scripts/bench_listener.py [--rounds 3] [--json out.json] [--small]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import skellysim_b200 as skb  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip()


def geometry(n_fib, n, ns, nbn, seed=0):
    """the node positions of scripts/bench_system_solve.py's system (the same draws in the same order)"""
    rng = np.random.default_rng(seed)
    c = rng.uniform(-4, 4, (n_fib, 1, 3))
    t = rng.normal(size=(n_fib, 1, 3))
    t /= np.linalg.norm(t, axis=2)[:, :, None]
    r_fib = (c + np.linspace(0, 1.0, n)[None, :, None] * t).reshape(-1, 3)
    sh = rng.normal(size=(ns, 3))
    sh /= np.linalg.norm(sh, axis=1)[:, None]
    i = np.arange(nbn)
    z = 1.0 - (2 * i + 1) / nbn
    th = np.pi * (3.0 - np.sqrt(5.0)) * i
    e = np.stack([np.sqrt(1 - z * z) * np.cos(th), np.sqrt(1 - z * z) * np.sin(th), z], axis=1)
    return r_fib, (6.0 * sh, -sh), (0.5 * e, e)


def timed(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def profile_split(torch, fn, out_dir):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t_wall, _ = timed(torch, fn)
    split = {"pair_sum_ms": 0.0, "listener_ms": 0.0, "other_ms": 0.0}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        ms = ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
        name = ev.name
        if "pair" in name or "reduce" in name or "pack" in name:
            split["pair_sum_ms"] += ms
        elif "line_" in name or "interior_replace" in name:
            split["listener_ms"] += ms
        else:  # the add-ons of the flow, copies and sets
            split["other_ms"] += ms
    busy = sum(split.values())
    split.update(wall_ms=t_wall * 1e3, gaps_ms=t_wall * 1e3 - busy)
    prof.export_chrome_trace(os.path.join(out_dir, "bench_listener_trace.json"))
    return {k: round(v, 3) for k, v in split.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--small", action="store_true")
    ap.add_argument("--trace-dir", default=tempfile.gettempdir(), help="where the profiler's trace is written")
    a = ap.parse_args()
    import torch
    import streamline_reference as sl
    if not torch.cuda.is_available():
        raise SystemExit("bench_listener.py needs a GPU")
    shape = (40, 32, 200, 100) if a.small else (3000, 32, 6000, 400)
    n_stream, n_vortex, n_host = (32, 8, 4) if a.small else (1024, 256, 16)
    r_fib, shell, body = geometry(*shape)
    rng = np.random.default_rng(1)
    ff, sd, bd = (rng.uniform(-1, 1, (len(r_fib), 3)), rng.uniform(-1, 1, (shape[2], 3)) * 0.1,
                  rng.uniform(-1, 1, (shape[3], 3)) * 0.1)
    ft = rng.uniform(-1, 1, (1, 6))
    d = rng.normal(size=(n_stream, 3))
    x0 = 4.0 * d / np.linalg.norm(d, axis=1)[:, None] * rng.uniform(0, 1, (n_stream, 1)) ** (1 / 3)
    eta = 1.0
    out = dict(card=card(), shape=dict(fibers=shape[0], nodes=shape[1], periphery=shape[2], body_nodes=shape[3]),
               strengths="seeded random, C3 size", lines=dict(streamlines=n_stream, vortexlines=n_vortex,
                                                              host_pattern=n_host))
    with skb.Flow(0) as fl:
        fl.set_fibers(r_fib, [shape[1]] * shape[0], [1.0] * shape[0])
        fl.set_periphery(*shell)
        fl.set_bodies(body[0], body[1], np.zeros((1, 3)))
        # kind 0: no interior test, so that (c)'s velocity_at_targets is the same function
        fl.set_listener_frame(ff, sd, bd, ft, np.zeros((1, 6)), [0], np.ones((1, 3)), eta)

        def host_velocity(p):
            return fl.velocity_at_targets(p, ff, sd, bd, ft, eta)

        arms = {"a": lambda: fl.streamlines(x0), "b": lambda: fl.vortexlines(x0[:n_vortex]),
                "c": lambda: sl.lines(host_velocity, x0[:n_host], max_points=1000)}  # the device's default cap
        for f in arms.values():  # warm every shape
            f()
        times = {k: [] for k in arms}
        res = {}
        for _ in range(a.rounds):
            for k, f in arms.items():
                dt, res[k] = timed(torch, f)
                times[k].append(dt)
        per = {"a": n_stream, "b": n_vortex, "c": n_host}
        out["per_line_ms"] = {k: dict(median=1e3 * float(np.median(v)) / per[k], min=1e3 * min(v) / per[k],
                                      max=1e3 * max(v) / per[k]) for k, v in times.items()}
        out["speedup_streamline_per_line"] = out["per_line_ms"]["c"]["median"] / out["per_line_ms"]["a"]["median"]
        pts = [len(l["time"]) for l in res["a"]]
        out["points_per_streamline"] = dict(mean=float(np.mean(pts)), max=int(max(pts)))
        out["statuses_a"] = {str(s): sum(1 for l in res["a"] if l["status"] == s)
                             for s in {l["status"] for l in res["a"]}}
        agree = dict(same_counts=0, same_status=0, max_dx=0.0)
        for g, e in zip(res["a"][:n_host], res["c"]):
            agree["same_status"] += g["status"] == e["status"]
            if len(g["time"]) == len(e["time"]):
                agree["same_counts"] += 1
                agree["max_dx"] = max(agree["max_dx"], float(np.abs(g["x"] - e["x"]).max()))
        out["agreement_a_vs_c"] = agree
        os.makedirs(a.trace_dir, exist_ok=True)
        out["profile_a"] = profile_split(torch, arms["a"], a.trace_dir)
        st = fl.stats()
        out["launches_last_call"] = st["launches"]
    print(json.dumps(out))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

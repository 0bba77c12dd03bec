"""Cost of the whole-vector operator over several devices (skb_mflow_apply_system_matvec, include/skelly_b200_flow.h)
against the partial operator skb_mflow_apply_matvec and the flow matvec skb_mflow_matvec on the same shape.

C3 (3000 fibers x 32 nodes, 6000 periphery nodes) with 1 body x 400 nodes and 200 fibers bound to it, the shape of
scripts/bench_system_matvec.py.  Per device list the three calls alternate, one of each per round: the system call forms
the links, the bodies' link forces (exchanged through the group window) and the body rows on the devices; the partial
call is given the link conditions and the bodies' forces and torques of the same x, computed beforehand on the host by
tests/system_reference.py (BodyContainer::calculate_link_conditions restated in numpy); the flow matvec takes the
strengths of the same x.  As a check that the system call and the partial call do the same work, the largest
relative difference of their fiber and periphery rows is reported (rounding only).
Reported per call: device_ms (skb_mflow_last_stats: CUDA events around each member's work, the slowest member, copies
excluded) and wall_ms (the host call, copies included), as medians with [min, max]; and the launches per call.  The
card's name and power limit are printed by the same run.  Needs a GPU; there is no CPU path.

    python scripts/bench_mflow_system.py [--reps 20] [--warmup 3] [--devices 0 / 0,0 / ...] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import skellysim_b200 as skb  # noqa: E402
from skellysim_b200 import capi  # noqa: E402
import system_reference as sr  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip()


def c3_shape(rng):
    n_fib, n, ns, nbn, n_bound = 3000, 32, 6000, 400, 200
    L = 1.0
    c = rng.uniform(-4, 4, (n_fib, 1, 3))
    t = rng.normal(size=(n_fib, 1, 3))
    t /= np.linalg.norm(t, axis=2)[:, :, None]
    r_fib = (c + np.linspace(0, L, n)[None, :, None] * t).reshape(-1, 3)
    sh = rng.normal(size=(ns, 3))
    sh /= np.linalg.norm(sh, axis=1)[:, None]
    e = rng.normal(size=(nbn, 3))
    e /= np.linalg.norm(e, axis=1)[:, None]
    body = np.full(n_fib, -1)
    body[rng.choice(n_fib, n_bound, replace=False)] = 0
    D = rng.normal(size=(n, n))
    return dict(n_fib=n_fib, n=n, ns=ns, nbn=nbn, L=L, r_fib=r_fib, sh=sh, r_b=0.5 * e, n_b=e, body=body, D=D,
                P=rng.normal(size=(4 * n - 14, 4 * n)), F=rng.normal(size=(3 * n, 4 * n)) / n,
                w=rng.uniform(0.5, 1.5, nbn), exyz=[rng.normal(size=(nbn, 3)) for _ in range(3)],
                site=0.5 * e[rng.integers(0, nbn, n_fib)], E=rng.uniform(0.5, 2.0, n_fib),
                M=rng.normal(size=(3 * ns, 3 * ns)) / np.sqrt(3 * ns))


def run(devs, s, reps, warmup, rng):
    n_fib, n, ns, nbn = s["n_fib"], s["n"], s["ns"], s["nbn"]
    nf = n_fib * n
    with skb.MultiFlow(devs) as mf:
        mf.set_fibers(s["r_fib"], [n] * n_fib, [s["L"]] * n_fib)
        mf.set_periphery(6.0 * s["sh"], -s["sh"])
        mf.set_bodies(s["r_b"], s["n_b"], np.zeros((1, 3)))
        mf.set_fiber_class(n, s["D"], s["P"])
        mf.set_fiber_class_derivatives(n, s["D"], s["D"], s["D"])
        A = np.broadcast_to(np.eye(4 * n), (n_fib, 4 * n, 4 * n))
        F = np.broadcast_to(s["F"], (n_fib, 3 * n, 4 * n))
        mf.set_fiber_operators(list(A), list(F), np.tile([1.0, 0.0, 0.0], (nf, 1)), [s["L"]] * n_fib, [0] * n_fib)
        mf.set_body_operators([nbn], s["w"], *s["exyz"])
        mf.set_fiber_links(s["body"], s["site"], s["E"])
        mf.set_dense(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, s["M"])
        x = rng.normal(size=mf.solution_size())
        x_f, x_s, x_b = x[:4 * nf], x[4 * nf:4 * nf + 3 * ns].reshape(ns, 3), x[4 * nf + 3 * ns:]
        dens = x_b[:3 * nbn].reshape(nbn, 3)
        link, ft = sr.link_conditions(dict(n_nodes=[n] * n_fib, lengths=[s["L"]] * n_fib),
                                      dict(xs=np.tile([1.0, 0.0, 0.0], (nf, 1)), D_2_0={n: s["D"]}, D_3_0={n: s["D"]}),
                                      dict(body=s["body"], site=s["site"], rigidity=s["E"]),
                                      dict(centers=np.zeros((1, 3)), n_nodes=[nbn]), x_f, x_b)
        out = {}

        def system():
            out["system"] = mf.apply_system_matvec(x, 1.0)

        def existing():
            out["existing"] = mf.apply_matvec(x_f, x_s, dens, ft, 1.0, link)

        def flow():
            out["matvec"] = mf.matvec(x_f[:3 * nf].reshape(nf, 3), x_s, dens, ft, 1.0)

        def timed(fn):
            t0 = time.perf_counter()
            fn()
            wall = (time.perf_counter() - t0) * 1e3
            st = mf.stats()
            return st["device_ms"], wall, st["launches"]

        for _ in range(warmup):
            system()
            existing()
            flow()
        t = {"system": [], "existing": [], "matvec": []}
        for _ in range(reps):  # alternating, one call of each per round
            t["system"].append(timed(system))
            t["existing"].append(timed(existing))
            t["matvec"].append(timed(flow))
    r_f, r_s, _ = out["existing"]  # the last call of each
    got = out["system"]
    rel = lambda a, b: float(np.abs(a - b).max() / np.abs(b).max())
    out = dict(devices=devs, check_fiber_rows_rel=rel(got[:4 * nf], r_f),
               check_shell_rows_rel=rel(got[4 * nf:4 * nf + 3 * ns], r_s.reshape(-1)))
    for k, v in t.items():
        v = np.array(v)
        for j, name in ((0, "device_ms"), (1, "wall_ms")):
            out[f"{k}_{name}"] = float(np.median(v[:, j]))
            out[f"{k}_{name}_spread"] = [float(v[:, j].min()), float(v[:, j].max())]
        out[f"{k}_launches"] = int(v[-1, 2])
    ds = np.array(t["system"])[:, 0] - np.array(t["existing"])[:, 0]
    out["diff_device_ms"] = float(np.median(ds))
    out["diff_device_ms_spread"] = [float(ds.min()), float(ds.max())]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--devices", nargs="*", default=None, help="device lists, e.g. 0 0,0 0,1")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if capi.device_count() == 0:
        raise SystemExit("bench_mflow_system.py needs a GPU")
    if a.devices:
        lists = [[int(d) for d in s.split(",")] for s in a.devices]
    else:
        lists = [[0], [0, 0]] + [list(range(k)) for k in (2, 4, 8) if capi.device_count() >= k]
    s = c3_shape(np.random.default_rng(0))
    out = dict(card=card(), case="C3 + 1 body x 400 nodes, 200 bound fibers",
               runs=[run(d, s, a.reps, a.warmup, np.random.default_rng(1)) for d in lists])
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

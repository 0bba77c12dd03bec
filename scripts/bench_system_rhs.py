"""Cost of the system right-hand side on the device (skb_flow_build_system_rhs_device, include/skelly_b200_flow.h).

C3 (3000 fibers x 32 nodes, 6000 periphery nodes) with one 400-node body, 200 fibers bound to it, 8 point sources and a
linear background flow.  In alternating rounds, one call of each per round:
  (a) skb_flow_build_system_rhs_device                         CUDA events around the call
  (b) skb_flow_apply_system_matvec_device on the same system   CUDA events, for scale
  (c) the composition available without it: skb_flow_matvec(f_ext, 0, 0, F_T) (downloads v_all), the point sources and
      the background on the host, skb_flow_build_fiber_rhs (uploads the fiber rows again), the negation of the shell and
      body rows on the host                                    host wall time, ending in a synchronise
Reports medians and min / max spreads, launches per call, and the largest difference between (a) and (c).  The card's
name and power limit are read by the same run.  Needs a GPU; there is no CPU path.

    python scripts/bench_system_rhs.py [--reps 15] [--warmup 3] [--json out.json]
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

import skellysim_b200 as skb  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip()


def event_ms(torch, fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def host_sources(r, pts, pf, pt, comp, scale, uni, eta):
    """psc.flow + bs.flow at r on the host (point_source.cpp:16-54, background_source.cpp:15-24; no target is within
    the regularisation radius of a point here)"""
    v = np.zeros_like(r)
    for p, f in zip(pts, pf):
        d = p - r
        dr = np.linalg.norm(d, axis=1)
        v += (f / dr[:, None] + d * ((d @ f) / dr**3)[:, None]) / (8 * np.pi * eta)
    for p, t in zip(pts, pt):
        d = r - p
        dr = np.linalg.norm(d, axis=1)
        v += np.cross(t, d) / dr[:, None] ** 3 / (8 * np.pi * eta)
    return v + uni[None, :] + r[:, comp] * scale[None, :]


def run(torch, reps, warmup):
    rng = np.random.default_rng(0)
    n_fib, n, ns, nbn, n_bound, eta, dt = 3000, 32, 6000, 400, 200, 1.0, 1e-3
    L = 1.0
    c = rng.uniform(-4, 4, (n_fib, 1, 3))
    t = rng.normal(size=(n_fib, 1, 3))
    t /= np.linalg.norm(t, axis=2)[:, :, None]
    r_fib = (c + np.linspace(0, L, n)[None, :, None] * t).reshape(-1, 3)
    sh = rng.normal(size=(ns, 3))
    sh /= np.linalg.norm(sh, axis=1)[:, None]
    e = rng.normal(size=(nbn, 3))
    e /= np.linalg.norm(e, axis=1)[:, None]
    r_b = 0.5 * e
    nf = n_fib * n
    pts, pf, pt = rng.uniform(-5, 5, (8, 3)), rng.normal(size=(8, 3)), rng.normal(size=(8, 3))
    comp, scale, uni = [1, 0, 2], np.array([0.1, -0.05, 0.0]), np.array([0.2, 0.0, -0.1])
    params = (np.full(n_fib, L), 2.5e-3, 0.0125, 500.0, 1.0, np.arange(n_fib) % 2, 0)
    f_ext = rng.uniform(-1, 1, (nf, 3))
    ft = rng.uniform(-1, 1, (1, 6))
    fs, vg = rng.uniform(-1, 1, n_fib), rng.uniform(-1, 1, n_fib)
    dev = torch.device("cuda", 0)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        fl.set_fibers(r_fib, [n] * n_fib, [L] * n_fib)
        fl.set_periphery(6.0 * sh, -sh)
        fl.set_bodies(r_b, e, np.zeros((1, 3)))
        D = rng.normal(size=(n, n)) / n
        fl.set_fiber_class(n, D, rng.normal(size=(4 * n - 14, 4 * n)) / n)
        fl.set_fiber_class_derivatives(n, D, D, D)
        A = np.ascontiguousarray(np.broadcast_to(np.eye(4 * n), (n_fib, 4 * n, 4 * n)))
        F = np.ascontiguousarray(np.broadcast_to(rng.normal(size=(3 * n, 4 * n)) / n, (n_fib, 3 * n, 4 * n)))
        fl.set_fiber_operators(A, F, np.tile([1.0, 0.0, 0.0], (nf, 1)), [L] * n_fib, [0] * n_fib)
        fl.set_body_operators([nbn], rng.uniform(0.5, 1.5, nbn), *(rng.normal(size=(nbn, 3)) for _ in range(3)))
        body = np.full(n_fib, -1)
        body[rng.choice(n_fib, n_bound, replace=False)] = 0
        fl.set_fiber_links(body, r_b[rng.integers(0, nbn, n_fib)], rng.uniform(0.5, 2.0, n_fib))
        M = rng.normal(size=(3 * ns, 3 * ns)) / np.sqrt(3 * ns)
        dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, M)
        del M
        fl.set_point_sources(pts, pf, pt)
        fl.set_background(comp, scale, uni)
        n_sol = fl.solution_size()
        x = torch.from_numpy(rng.normal(size=n_sol)).to(dev)
        res = torch.zeros_like(x)
        rhs = torch.zeros_like(x)
        d_f = torch.from_numpy(f_ext).to(dev)
        d_F, d_T = torch.from_numpy(ft[:, :3].copy()).to(dev), torch.from_numpy(ft[:, 3:].copy()).to(dev)
        st = torch.cuda.current_stream().cuda_stream
        r_nodes = np.concatenate([r_fib, 6.0 * sh, r_b])
        zs, zb = np.zeros((ns, 3)), np.zeros((nbn, 3))

        def device_rhs():
            fl.build_system_rhs_device(*params, dt, eta, d_f.data_ptr(), d_F.data_ptr(), d_T.data_ptr(),
                                       rhs.data_ptr(), v_growth=vg, force_scale=fs, stream=st)

        def matvec():
            fl.apply_system_matvec_device(dn, x.data_ptr(), eta, res.data_ptr(), st)

        def composed():
            v = fl.matvec(f_ext, zs, zb, ft, eta)
            v += host_sources(r_nodes, pts, pf, pt, comp, scale, uni, eta)
            fr = fl.build_fiber_rhs(*params, dt, eta, v_on_fibers=v[:nf], f_external=f_ext, v_growth=vg,
                                    force_scale=fs)
            return np.concatenate([fr, -v[nf:nf + ns].reshape(-1), -v[nf + ns:].reshape(-1), np.zeros(6)])

        def composed_timed():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = composed()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3, out

        for _ in range(warmup):
            device_rhs()
            matvec()
            composed_timed()
        torch.cuda.synchronize()
        launches = {}
        device_rhs()
        launches["rhs"] = fl.stats()["launches"]
        matvec()
        launches["system_matvec"] = fl.stats()["launches"]
        ta, tb, tc = [], [], []
        for _ in range(reps):  # alternating, one call of each per round
            ta.append(event_ms(torch, device_rhs))
            tb.append(event_ms(torch, matvec))
            ms, comp_out = composed_timed()
            tc.append(ms)
        got = rhs.cpu().numpy()
    ta, tb, tc = np.array(ta), np.array(tb), np.array(tc)
    diff = float(np.abs(got - comp_out).max() / np.abs(comp_out).max())
    spread = lambda a: [float(a.min()), float(a.max())]
    return dict(case="C3 + 1 body x 400 nodes, 200 bound fibers, 8 point sources, background flow",
                rhs_device_ms=float(np.median(ta)), rhs_device_ms_spread=spread(ta),
                system_matvec_ms=float(np.median(tb)), system_matvec_ms_spread=spread(tb),
                composed_wall_ms=float(np.median(tc)), composed_wall_ms_spread=spread(tc),
                launches_rhs=launches["rhs"], launches_system_matvec=launches["system_matvec"],
                rel_max_diff_rhs_vs_composed=diff, reps=int(reps))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_system_rhs.py needs a GPU")
    out = dict(card=card(), rhs=run(torch, a.reps, a.warmup))
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

"""Cost of the body block and the fiber-body links on the device (skb_flow_apply_system_matvec_device /
_preconditioner_device, include/skelly_b200_flow.h).

1. C3 (3000 fibers x 32 nodes, 6000 periphery nodes, 1 body x 400 nodes) with 200 fibers bound to the body: the
   whole-vector A x against skb_flow_apply_matvec_device on the same inputs (the links and the body rows given as
   zeros / passed through), alternating in one run, CUDA events around each call; the difference and the added launches.
2. The body preconditioner's GEMV at 1 body x 2000 nodes (A_^-1 of 6006 x 6006, 289 MB): bytes over kernel time
   against the H100 SXM data sheet's 3.35 TB/s.
The card's name and power limit are printed by the same run.  Needs a GPU; there is no CPU path.

    python scripts/bench_system_matvec.py [--reps 20] [--warmup 3] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import skellysim_b200 as skb  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data sheet


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip()


def timed(torch, fn, reps):
    """per-call milliseconds of fn() over reps calls (CUDA events on the current stream)"""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def sphere(n, radius, center, rng):
    e = rng.normal(size=(n, 3))
    e /= np.linalg.norm(e, axis=1)[:, None]
    return center + radius * e, e


def c3_matvec(torch, reps, warmup):
    rng = np.random.default_rng(0)
    n_fib, n, ns, nbn, n_bound = 3000, 32, 6000, 400, 200
    L = 1.0
    c = rng.uniform(-4, 4, (n_fib, 1, 3))
    t = rng.normal(size=(n_fib, 1, 3))
    t /= np.linalg.norm(t, axis=2)[:, :, None]
    r_fib = (c + np.linspace(0, L, n)[None, :, None] * t).reshape(-1, 3)
    sh = rng.normal(size=(ns, 3))
    sh /= np.linalg.norm(sh, axis=1)[:, None]
    center = np.zeros(3)
    r_b, n_b = sphere(nbn, 0.5, center, rng)
    nf = n_fib * n
    dev = torch.device("cuda", 0)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        fl.set_fibers(r_fib, [n] * n_fib, [L] * n_fib)
        fl.set_periphery(6.0 * sh, -sh)
        fl.set_bodies(r_b, n_b, center[None])
        D = rng.normal(size=(n, n))
        fl.set_fiber_class(n, D, rng.normal(size=(4 * n - 14, 4 * n)))
        fl.set_fiber_class_derivatives(n, D, D, D)
        A = np.ascontiguousarray(np.broadcast_to(np.eye(4 * n), (n_fib, 4 * n, 4 * n)))
        F = np.ascontiguousarray(np.broadcast_to(rng.normal(size=(3 * n, 4 * n)) / n, (n_fib, 3 * n, 4 * n)))
        fl.set_fiber_operators(A, F, np.tile([1.0, 0.0, 0.0], (nf, 1)), [L] * n_fib, [0] * n_fib)
        fl.set_body_operators([nbn], rng.uniform(0.5, 1.5, nbn), *(rng.normal(size=(nbn, 3)) for _ in range(3)))
        body = np.full(n_fib, -1)
        body[rng.choice(n_fib, n_bound, replace=False)] = 0
        fl.set_fiber_links(body, r_b[rng.integers(0, nbn, n_fib)], rng.uniform(0.5, 2.0, n_fib))  # sites on the surface
        M = rng.normal(size=(3 * ns, 3 * ns)) / np.sqrt(3 * ns)
        dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, M)
        del M
        n_sol = fl.solution_size()
        x = torch.from_numpy(rng.normal(size=n_sol)).to(dev)
        res = torch.zeros_like(x)
        x_f, x_s, x_b = x[:4 * nf], x[4 * nf:4 * nf + 3 * ns], x[4 * nf + 3 * ns:]
        dens = x_b[:3 * nbn].clone()
        zeros = torch.zeros(3, dtype=torch.float64, device=dev)
        link = torch.zeros(7 * n_fib, dtype=torch.float64, device=dev)
        r_f, r_s, v_b = (torch.zeros(k, dtype=torch.float64, device=dev) for k in (4 * nf, 3 * ns, 3 * nbn))
        st = torch.cuda.current_stream().cuda_stream

        def system():
            fl.apply_system_matvec_device(dn, x.data_ptr(), 1.0, res.data_ptr(), st)

        def existing():
            fl.apply_matvec_device(dn, x_f.data_ptr(), x_s.data_ptr(), dens.data_ptr(), zeros.data_ptr(),
                                   zeros.data_ptr(), link.data_ptr(), 1.0, r_f.data_ptr(), r_s.data_ptr(),
                                   v_b.data_ptr(), st)

        for _ in range(warmup):
            system()
            existing()
        torch.cuda.synchronize()
        launches = {}
        system()
        launches["system"] = fl.stats()["launches"]
        existing()
        launches["existing"] = fl.stats()["launches"]
        t_sys, t_old = [], []
        for _ in range(reps):  # alternating, one call of each per round
            t_sys.append(timed(torch, system, 1))
            t_old.append(timed(torch, existing, 1))
    t_sys, t_old = np.array(t_sys), np.array(t_old)
    return dict(case="C3 + 1 body x 400 nodes, 200 bound fibers", system_ms=float(np.median(t_sys)),
                existing_ms=float(np.median(t_old)), diff_ms=float(np.median(t_sys - t_old)),
                system_ms_spread=[float(t_sys.min()), float(t_sys.max())],
                existing_ms_spread=[float(t_old.min()), float(t_old.max())],
                launches_system=launches["system"], launches_existing=launches["existing"],
                added_launches=launches["system"] - launches["existing"])


def body_gemv(torch, reps, warmup):
    rng = np.random.default_rng(1)
    nbn = 2000
    m = 3 * nbn + 6
    r_b, n_b = sphere(nbn, 1.0, np.zeros(3), rng)
    dev = torch.device("cuda", 0)
    with skb.Flow(0) as fl:
        fl.set_fibers(np.zeros((0, 3)), [], [])
        fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_bodies(r_b, n_b, np.zeros((1, 3)))
        fl.set_fiber_operators([], [], np.zeros((0, 3)), [], [])
        fl.set_fiber_preconditioner([])
        A_inv = rng.normal(size=(m, m))
        fl.set_body_operators([nbn], np.ones(nbn), *(rng.normal(size=(nbn, 3)) for _ in range(3)), [A_inv])
        x = torch.from_numpy(rng.normal(size=m)).to(dev)
        y = torch.zeros_like(x)
        st = torch.cuda.current_stream().cuda_stream
        call = lambda: fl.apply_system_preconditioner_device(None, x.data_ptr(), y.data_ptr(), st)
        for _ in range(warmup):
            call()
        torch.cuda.synchronize()
        ms = timed(torch, call, reps)
        launches = fl.stats()["launches"]
        err = float(np.abs(y.cpu().numpy() - A_inv @ x.cpu().numpy()).max() / np.abs(A_inv @ x.cpu().numpy()).max())
    nbytes = 8.0 * m * m
    tbs = nbytes / (ms * 1e-3) / 1e12
    return dict(case="body preconditioner GEMV, 1 body x 2000 nodes", unknowns=m, bytes=nbytes, ms=ms, tb_s=tbs,
                share_of_3p35=tbs / HBM_TBS, launches=launches, rel_err_vs_numpy=err)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_system_matvec.py needs a GPU")
    out = dict(card=card(), matvec=c3_matvec(torch, a.reps, a.warmup), gemv=body_gemv(torch, 10 * a.reps, a.warmup))
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

"""Cost of the whole-system solve on the device (skb_flow_solve_system_device, include/skelly_b200_flow.h).

C3 (3000 fibers x 32 nodes) with the fiber operators and their inverse built on the device, 6000 periphery nodes with a
well-conditioned stand-in operator I + U V^T / 16 (rank 16) and its exact inverse by Woodbury (the host never inverts an
18 000^2 matrix), one 400-node sphere with its true operator and inverse and 200 fibers bound to it; the RHS built on
the device; solved at tol 1e-10.  In alternating rounds:
  (a) the device solve (skb_flow_solve_system_device)                                  host wall time, synchronised
  (b) tests/gmres_reference.py on the host over SystemOperator.apply / .apply_preconditioner: the composition a caller
      has without (a), the same algorithm and iterations                               host wall time
Reports the card's name and power limit (read by the same run), iterations, medians and min / max, time per iteration,
the share of (a) outside A and P^-1 (their CUDA-event time over the same number of applies), the orthogonalization
passes' bytes / time at k = 16, 100 and 300 basis vectors (24 k n bytes per Arnoldi step, share of 3.35 TB/s; None where
the estimate falls below its noise).  Needs a GPU; --small runs the construction at a tiny size.

    python scripts/bench_system_solve.py [--reps 3] [--json out.json] [--small]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import skellysim_b200 as skb  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip()


def system(n_fib, n, ns, nbn, n_bound, rank, seed=0):
    """the host arrays of the benchmark system"""
    import system_reference as sr
    from oracle.fiber_fd import compute_matrices
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
    R = 0.5
    r_b, w_b = R * e, np.full(nbn, 4 * np.pi * R * R / nbn)
    ex, ey, ez = sr.singularity_vectors(r_b, e, w_b)
    A_b = sr.body_operator(r_b, e, np.zeros(3), w_b, ex, ey, ez)
    U = rng.normal(size=(3 * ns, rank)) / np.sqrt(3 * ns)
    V = rng.normal(size=(3 * ns, rank)) / np.sqrt(3 * ns) / 16
    M = np.eye(3 * ns) + U @ V.T
    Minv = np.eye(3 * ns) - U @ np.linalg.solve(np.eye(rank) + V.T @ U, V.T)  # Woodbury
    body = np.full(n_fib, -1)
    body[:n_bound] = 0  # bound fibers precede the free ones
    site = r_fib.reshape(n_fib, n, 3)[:, 0]
    return dict(r_fib=r_fib, shell=(6.0 * sh, -sh), body=(r_b, e, w_b, ex, ey, ez, np.linalg.inv(A_b)), M=M,
                Minv=Minv, links=(body, site), mats=compute_matrices(n), n=n, n_fib=n_fib)


def run(torch, reps, small, tol=1e-10, eta=1.0, dt=1e-3):
    from gmres_reference import gmres
    from skellysim_b200.solver_hydro import SystemOperator
    shape = (40, 32, 200, 100, 10, 4) if small else (3000, 32, 6000, 400, 200, 16)
    s = system(*shape)
    n, n_fib = s["n"], s["n_fib"]
    dev = torch.device("cuda", 0)
    params = (np.full(n_fib, 1.0), 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)
    out = dict(card=card(), shape=dict(fibers=n_fib, nodes=n, periphery=shape[2], body_nodes=shape[3],
                                       bound=shape[4]), tol=tol)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        fl.set_fibers(s["r_fib"], [n] * n_fib, [1.0] * n_fib)
        fl.set_periphery(*s["shell"])
        r_b, e, w_b, ex, ey, ez, A_inv = s["body"]
        fl.set_bodies(r_b, e, np.zeros((1, 3)))
        m = s["mats"]
        fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
        fl.build_fiber_operators(*params, dt, eta)
        fl.set_body_operators([len(w_b)], w_b, ex, ey, ez, [A_inv])
        body, site = s["links"]
        fl.set_fiber_links(body, site, 2.5e-3)
        dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, s["M"])
        dn.set_matrix(skb.DENSE_M_INV, s["Minv"])
        del s
        op = SystemOperator(fl, dn, eta, dev)
        f_ext = torch.from_numpy(np.random.default_rng(1).uniform(-1, 1, (n_fib * n, 3))).to(dev)
        b = op.rhs(params, dt, f_external=f_ext)
        op.set_gmres(300)
        out["n"] = op.n
        x, info = op.solve(b, tol=tol)  # warm-up, and the iteration count
        torch.cuda.synchronize()
        k = info["iterations"]
        out["device"] = {key: info[key] for key in ("converged", "iterations", "restarts", "explicit_residual")}
        b_np = b.cpu().numpy()
        to = lambda v: torch.from_numpy(v).to(dev)
        A = lambda v: op.apply(to(v)).cpu().numpy()
        P = lambda v: op.apply_preconditioner(to(v)).cpu().numpy()
        t_dev, t_host = [], []
        for _ in range(reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            op.solve(b, tol=tol)
            torch.cuda.synchronize()
            t_dev.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            _, hinfo = gmres(A, P, b_np, tol=tol)
            t_host.append(time.perf_counter() - t0)
        out["host_iterations"] = hinfo["iterations"]
        # A and P^-1 alone, as many applies as the solve makes (k + cycle ends)
        applies = k + 2 * (info["restarts"] + 1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        z = torch.zeros_like(b)
        e0.record()
        for _ in range(applies):
            z = op.apply(op.apply_preconditioner(b)).clone()
        e1.record()
        e1.synchronize()
        ops_s = e0.elapsed_time(e1) / 1e3
        med = float(np.median(t_dev))
        out["solve_s"] = dict(median=med, min=min(t_dev), max=max(t_dev), per_iteration=med / max(k, 1),
                              outside_A_Pinv_share=max(0.0, 1 - ops_s / med))
        out["host_composition_s"] = dict(median=float(np.median(t_host)), min=min(t_host), max=max(t_host))
        # the orthogonalization passes alone at k basis vectors: 3 passes over V (k columns) per step
        out["orthogonalization"] = {}
        for kk in (16, 100, 300):
            t = ortho_time(torch, op, b, kk)
            byt = 24.0 * kk * op.n
            out["orthogonalization"][kk] = None if t is None else dict(
                ms_per_step=t * 1e3, TB_s=byt / t / 1e12, share_of_3_35=byt / t / 3.35e12)
    return out


def ortho_time(torch, op, b, k):
    """time per Arnoldi step at k basis vectors, less the time of the step's A and P^-1: a solve limited to k steps in
    one cycle (max_iters = k), its per-step time at the last steps estimated from two solves of k and k - 8 steps"""
    def solve_s(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        op.solve(b, tol=1e-300, num_blocks=300, max_iters=steps)
        torch.cuda.synchronize()
        return time.perf_counter() - t0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(8):
        op.apply(op.apply_preconditioner(b))
    e1.record()
    e1.synchronize()
    ops8 = e0.elapsed_time(e1) / 1e3
    d = min(solve_s(k) - solve_s(k - 8) for _ in range(2))
    return (d - ops8) / 8 if d > ops8 else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--small", action="store_true", help="a tiny system: construction and plumbing only")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        if a.small:
            s = system(40, 32, 200, 100, 10, 4)
            print(f"constructed the --small system ({s['r_fib'].shape[0]} fiber nodes); no GPU, nothing timed")
            return
        raise SystemExit("bench_system_solve.py needs a GPU")
    out = run(torch, a.reps, a.small)
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

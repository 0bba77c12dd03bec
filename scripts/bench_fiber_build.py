#!/usr/bin/env python
"""The per-fiber operators and their inverse built on the device (skb_flow_build_fiber_operators) against uploading
the same operators (GPU box): 3000 x 32 (BASELINE C3) and 2000 x 64 straight fibers, free ends, a random half hinged at
the plus end.  Prints one JSON line with the card's name and power limit.
usage: bench_fiber_build.py [reps=10]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import skellysim_b200 as skb  # noqa: E402
from skellysim_b200 import capi  # noqa: E402


def fiber_build_leg(local_rank=0, reps=10, n_checked=8):
    """skb_flow_build_fiber_operators: A_, force_operator_, xs_ and A_^-1 built on the device (update_derivatives,
    update_linear_operator, update_force_operator, apply_bc_rectangular's operator half, update_preconditioner) for
    straight fibers with free ends, a random half of them hinged at the plus end -- against uploading the same operators
    (skb_flow_set_fiber_operators + skb_flow_set_fiber_preconditioner of what the build made, read back).  Build time:
    the call's CUDA events (skb_flow_last_stats device_ms: its kernels; total_ms: with its table uploads) and the host
    clock around the call, warm, median of `reps`; kernel split from torch.profiler.  FLOP from shapes: the projection
    P_downsample_bc * A_ over P's non-zeros (2 (4n-14) n 4n per fiber) and Gauss-Jordan (2 (4n)^3 per fiber)."""
    from oracle import fiber_fd  # class matrices (host constants of the reference) and the sample check
    out = {}
    for n_fibers, n in ((3000, 32), (2000, 64)):
        fib, _, _, _ = bench.make_suspension(n_fibers, 0, seed=5, n_nodes=n)
        rng = np.random.default_rng([5, n])
        hinged = (rng.random(n_fibers) < 0.5).astype(np.int32)
        prm = dict(length_prev=1.0, bending_rigidity=2.5e-3, radius=0.0125, penalty_param=500.0, beta_tstep=1.0,
                   minus_clamped=0, plus_hinged=hinged)
        dt = 1e-2
        m = fiber_fd.compute_matrices(n)
        fl = skb.Flow(local_rank)
        fl.set_fibers(fib, np.full(n_fibers, n, dtype=np.int32), np.ones(n_fibers))
        fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_bodies(np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
        build = lambda: fl.build_fiber_operators(*prm.values(), dt, bench.ETA)
        for _ in range(2):
            build()
        wall, dev_ms, tot_ms = [], [], []
        for _ in range(reps):
            t0 = time.perf_counter()
            build()
            wall.append(1e3 * (time.perf_counter() - t0))
            st = fl.stats()
            dev_ms.append(st["device_ms"])
            tot_ms.append(st["total_ms"])
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                build()
        k_ms = {"fiber_assemble_kernel": 0.0, "fiber_inverse_kernel": 0.0}
        for e in prof.key_averages():
            for k in k_ms:
                if k in e.key:
                    k_ms[k] += e.device_time_total / 1e3 / 3  # (us over 3 builds)
        # the upload it replaces: the same operators from pageable host memory
        A = np.empty(n_fibers * 16 * n * n)
        F = np.empty(n_fibers * 12 * n * n)
        Ai = np.empty_like(A)
        xs = np.empty((n_fibers * n, 3))
        L = capi.library()
        capi._check(L.skb_flow_get_fiber_operators(fl._h, capi._p(A), capi._p(F), capi._p(xs), capi._p(Ai)))
        up_ops, up_inv = [], []
        for _ in range(3):
            t0 = time.perf_counter()
            fl.set_fiber_operators(A, F, xs, np.ones(n_fibers), hinged, colmajor=True)
            t1 = time.perf_counter()
            capi._check(L.skb_flow_set_fiber_preconditioner(fl._h, capi._p(Ai)))
            torch.cuda.synchronize()
            up_ops.append(1e3 * (t1 - t0))
            up_inv.append(1e3 * (time.perf_counter() - t1))
        # sample against the oracle (the straight fibers of bench.make_suspension have length 1 = length_prev)
        errs, resid = [], []
        for f in np.random.default_rng(9).choice(n_fibers, n_checked, replace=False):
            fo = fiber_fd.FiberOperators(fib[f * n:(f + 1) * n], 1.0, eta=bench.ETA, dt=dt, plus_pinned=bool(hinged[f]))
            Af = A[f * 16 * n * n:(f + 1) * 16 * n * n].reshape(4 * n, 4 * n).T
            Ff = F[f * 12 * n * n:(f + 1) * 12 * n * n].reshape(4 * n, 3 * n).T
            Xf = Ai[f * 16 * n * n:(f + 1) * 16 * n * n].reshape(4 * n, 4 * n).T
            errs += [np.abs(Af - fo.A).max() / np.abs(fo.A).max(),
                     np.abs(Ff - fo.force_operator).max() / np.abs(fo.force_operator).max(),
                     np.abs(xs[f * n:(f + 1) * n] - fo.xs).max() / np.abs(fo.xs).max()]
            resid.append(np.linalg.norm(Af @ Xf - np.eye(4 * n)) / (np.linalg.norm(Af) * np.linalg.norm(Xf)))
        fl.close()
        flop_asm = n_fibers * 2.0 * (4 * n - 14) * n * 4 * n
        flop_inv = n_fibers * 2.0 * (4 * n) ** 3
        ka, ki = k_ms["fiber_assemble_kernel"], k_ms["fiber_inverse_kernel"]
        key = f"{n_fibers}x{n}"
        out[key] = {
            "build_ms": float(np.median(dev_ms)), "build_total_ms": float(np.median(tot_ms)),
            "build_wall_ms": float(np.median(wall)), "assemble_kernel_ms": ka, "inverse_kernel_ms": ki,
            "gflop_assemble": flop_asm / 1e9, "gflop_inverse": flop_inv / 1e9,
            "tflops_assemble": flop_asm / (ka * 1e-3) / 1e12 if ka else None,
            "tflops_inverse": flop_inv / (ki * 1e-3) / 1e12 if ki else None,
            "frac_of_nominal_fp64_assemble": flop_asm / (ka * 1e-3) / 1e12 / bench.NOMINAL_FP64_TFLOPS if ka else None,
            "frac_of_nominal_fp64_inverse": flop_inv / (ki * 1e-3) / 1e12 / bench.NOMINAL_FP64_TFLOPS if ki else None,
            "upload_operators_ms": float(np.median(up_ops)), "upload_inverse_ms": float(np.median(up_inv)),
            "operator_bytes": int(A.nbytes + F.nbytes), "inverse_bytes": int(Ai.nbytes),
            "sample_max_rel_err_vs_oracle": float(max(errs)), "sample_max_inverse_residual": float(max(resid)),
            "n_checked": int(n_checked)}
        del A, F, Ai
    out["note"] = ("build_ms: CUDA events around the build's kernels (skb_flow_last_stats); build_wall_ms: host clock "
                   "around the whole call; upload_*: host clock around skb_flow_set_fiber_operators / "
                   "skb_flow_set_fiber_preconditioner of the same operators (pageable host memory); kernel split: "
                   "torch.profiler, mean of 3 builds; fp64 peak: nominal 33.5 TFLOP/s (H100 SXM)")
    return out


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    if not torch.cuda.is_available():
        raise SystemExit("bench_fiber_build.py needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    out = fiber_build_leg(0, reps=reps)
    out["gpu"] = card
    print(json.dumps(out))


if __name__ == "__main__":
    main()

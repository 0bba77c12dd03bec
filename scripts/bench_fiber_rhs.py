#!/usr/bin/env python
"""The fiber block of the RHS formed on the device (skb_flow_build_fiber_rhs), GPU box: 3000 x 32 (BASELINE C3) and
2000 x 64 straight fibers, length_prev 2 % off length_, random flow and external force at the nodes, random growth
velocities and motor force scales, free ends and a random half hinged at the plus end.  Prints one JSON line with the
card's name and power limit, read in the same run.
usage: bench_fiber_rhs.py [reps=20]"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # fiber_rhs_reference: the sample check
import bench  # noqa: E402
import skellysim_b200 as skb  # noqa: E402

U = 2.0 ** -53


def fiber_rhs_leg(local_rank=0, reps=20, n_checked=6):
    """skb_flow_build_fiber_rhs, warm, median of `reps`: device_ms (CUDA events around the kernel, skb_flow_last_stats),
    total_ms (with the uploads of v_on_fibers, f_external and the per-fiber tables and the download of the RHS), the
    host clock around the call, and the kernel alone from torch.profiler.  Bytes from shapes: host -> device (two
    3 x N_f inputs and 120 bytes of tables per fiber), device -> host (4 N_f), and the kernel's compulsory global
    traffic (positions, the two inputs, the output; the class matrices stay in L2).  A sample of fibers is held to the
    long-double reference (tests/fiber_rhs_reference.py): max |dev - ext| / (u S)."""
    from fiber_rhs_reference import fiber_rhs  # the sample check
    from oracle import fiber_fd  # class matrices (host constants of the reference) and the sample check
    out = {}
    for n_fibers, n in ((3000, 32), (2000, 64)):
        fib, _, _, _ = bench.make_suspension(n_fibers, 0, seed=5, n_nodes=n)
        rng = np.random.default_rng([7, n])
        nf = n_fibers * n
        hinged = (rng.random(n_fibers) < 0.5).astype(np.int32)
        prm = dict(length_prev=np.full(n_fibers, 0.98), bending_rigidity=2.5e-3, radius=0.0125, penalty_param=500.0,
                   beta_tstep=1.0, minus_clamped=0, plus_hinged=hinged)
        inp = dict(v_on_fibers=rng.uniform(-1, 1, (nf, 3)), f_external=rng.uniform(-1, 1, (nf, 3)),
                   v_growth=rng.uniform(-0.1, 0.1, n_fibers), force_scale=rng.uniform(-1, 1, n_fibers))
        dt = 1e-2
        m = fiber_fd.compute_matrices(n)
        fl = skb.Flow(local_rank)
        fl.set_fibers(fib, np.full(n_fibers, n, dtype=np.int32), np.ones(n_fibers))
        fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_bodies(np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
        call = lambda: fl.build_fiber_rhs(*prm.values(), dt, bench.ETA, **inp)
        for _ in range(3):
            rhs = call()
        wall, dev_ms, tot_ms = [], [], []
        for _ in range(reps):
            t0 = time.perf_counter()
            call()
            wall.append(1e3 * (time.perf_counter() - t0))
            st = fl.stats()
            dev_ms.append(st["device_ms"])
            tot_ms.append(st["total_ms"])
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                call()
        k_ms = sum(e.device_time_total for e in prof.key_averages() if "fiber_rhs_kernel" in e.key) / 1e3 / 5
        fl.close()
        # the sample against the long-double oracle (straight fibers of bench.make_suspension: length_ 1)
        worst = 0.0
        for f in np.random.default_rng(9).choice(n_fibers, n_checked, replace=False):
            sl = slice(f * n, (f + 1) * n)
            kw = dict(v=inp["v_on_fibers"][sl], f_external=inp["f_external"][sl],
                      force_scale=inp["force_scale"][f], v_growth=inp["v_growth"][f])
            ext, S = (fiber_rhs(fiber_fd.FiberOperators(fib[sl], 1.0, eta=bench.ETA, dt=dt, length_prev=0.98,
                                                        plus_pinned=bool(hinged[f]), **d), **kw)
                      for d in (dict(dtype=np.longdouble), dict(absolute=True)))
            d = np.abs(rhs[4 * f * n:4 * (f + 1) * n].astype(np.longdouble) - ext).astype(np.float64)
            with np.errstate(divide="ignore", invalid="ignore"):
                worst = max(worst, float(np.max(np.where(S > 0, d / (U * S), np.where(d == 0, 0.0, np.inf)))))
        out[f"{n_fibers}x{n}"] = {
            "device_ms": float(np.median(dev_ms)), "total_ms": float(np.median(tot_ms)),
            "wall_ms": float(np.median(wall)), "kernel_ms_profiler": k_ms,
            "h2d_bytes": int(2 * nf * 24 + n_fibers * 120), "d2h_bytes": int(nf * 32),
            "kernel_global_bytes": int(nf * (3 * 24 + 32) + n_fibers * 120),
            "sample_max_err_over_uS": worst, "n_checked": int(n_checked)}
    out["note"] = ("device_ms: CUDA events around the RHS kernel (skb_flow_last_stats); total_ms: with the uploads of "
                   "the inputs and per-fiber tables and the download of the RHS (pageable host memory); wall_ms: host "
                   "clock around the call; kernel_ms_profiler: torch.profiler, mean of 5 calls; "
                   "sample_max_err_over_uS: max |dev - ext| / (u S) over the sampled fibers (tests hold it to <= 8)")
    return out


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    if not torch.cuda.is_available():
        raise SystemExit("bench_fiber_rhs.py needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    out = fiber_rhs_leg(0, reps=reps)
    out["gpu"] = card
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Per-call device time of the rank-per-GPU whole-vector calls (skb_flow_group_apply_system_matvec_device,
_apply_system_preconditioner_device, _build_system_rhs_device, include/skelly_b200_flow.h) against skb_mflow on the same
device list and the single-device _device calls.

C3 (3000 fibers x 32 nodes, 6000 periphery nodes) with 1 body x 400 nodes and 200 fibers bound to it, the shape of
scripts/bench_mflow_system.py.  Forms, one call of each per round, alternating:
  group   n members connected by skb_flow_group_connect, each driven by its own host thread on its own stream; device
          time = CUDA events around each member's call, the slowest member
  mflow   skb_mflow on the same device list (skb_mflow_last_stats: the slowest member, copies excluded)
  single  one flow on device 0, the whole vector (CUDA events around the _device call)
Reported per call: the median and [min, max] of the device time over the rounds, and the launches per call.  The card's
name and power limit are printed by the same run.  Needs a GPU; there is no CPU path.

    python scripts/bench_group_system.py [--reps 15] [--warmup 3] [--devices 0,0 0,1] [--json out.json]
"""
import argparse
import json
import os
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import skellysim_b200 as skb  # noqa: E402
from skellysim_b200 import capi, distributed  # noqa: E402
from bench_mflow_system import c3_shape, card  # noqa: E402

DT, ETA = 1e-3, 1.0
CALLS = ("matvec", "precondition", "rhs")


def geometry(fl, s):
    fl.set_fibers(s["r_fib"], [s["n"]] * s["n_fib"], [s["L"]] * s["n_fib"])
    fl.set_periphery(6.0 * s["sh"], -s["sh"])
    fl.set_bodies(s["r_b"], s["n_b"], np.zeros((1, 3)))


def operators(fl, s, f0, f1, body_ops, links):
    n, nf = s["n"], (f1 - f0) * s["n"]
    fl.set_fiber_class(n, s["D"], s["P"])
    fl.set_fiber_class_derivatives(n, s["D"], s["D"], s["D"])
    A = [np.eye(4 * n)] * (f1 - f0)
    fl.set_fiber_operators(A, [s["F"]] * (f1 - f0), np.tile([1.0, 0.0, 0.0], (nf, 1)), [s["L"]] * (f1 - f0),
                           [0] * (f1 - f0))
    fl.set_fiber_preconditioner(A)
    body_ops(s["nbn"], s["w"], *s["exyz"], [s["Ainv_b"]])
    links(s["body"][f0:f1], s["site"][f0:f1], s["E"][f0:f1])


def params(s, k):
    return (np.full(k, s["L"]), 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)


def summary(ts):
    v = np.array(ts)
    return dict(device_ms=float(np.median(v[:, 0])), device_ms_spread=[float(v[:, 0].min()), float(v[:, 0].max())],
                launches=int(v[-1, 1]))


def run_group(devs, s, x, reps, warmup):
    import torch
    n = len(devs)
    fn = [s["n"]] * s["n_fib"]
    parts = [capi.partition_query(fn, s["ns"], s["nbn"], n, g) for g in range(n)]
    flows = [skb.Flow(d) for d in devs]
    dense = []
    try:
        for g, fl in enumerate(flows):
            geometry(fl, s)
            fl.set_target_ranges(*parts[g])
            fl.group_init(g, n)
        for g, fl in enumerate(flows):
            for h in range(n):
                if h != g:
                    fl.group_connect(h, flows[h])
        ops = []
        for g, fl in enumerate(flows):
            fl.group_warmup()
            f0, f1, s0, s1 = parts[g][:4]
            operators(fl, s, f0, f1, lambda nb, w, ex, ey, ez, ai: fl.group_set_body_operators([nb], w, ex, ey, ez, ai),
                      fl.group_set_fiber_links)
            dm, dp = skb.Dense(device_ids=[devs[g]]), skb.Dense(device_ids=[devs[g]])
            dm.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, s["M"][3 * s0:3 * s1])
            dp.set_matrix(skb.DENSE_M_INV, s["M"][3 * s0:3 * s1])
            dense += [dm, dp]
            ops.append(distributed.RankSystemOperator(fl, dm, dp, parts[g], fn, s["ns"], [s["nbn"]], ETA,
                                                      torch.device("cuda", devs[g])))
        xs = [torch.from_numpy(x[o.local_rows]).to(f"cuda:{d}") for o, d in zip(ops, devs)]
        streams = [torch.cuda.Stream(device=d) for d in devs]
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in devs]

        def one(call):
            def fn_(g):
                f0, f1 = parts[g][:2]
                with torch.cuda.stream(streams[g]):
                    ev[g][0].record()
                    if call == "matvec":
                        ops[g].apply(xs[g])
                    elif call == "precondition":
                        ops[g].apply_preconditioner(xs[g])
                    else:
                        ops[g].rhs(params(s, f1 - f0), DT)
                    ev[g][1].record()
                streams[g].synchronize()
            th = [threading.Thread(target=fn_, args=(g,)) for g in range(n)]
            for t in th:
                t.start()
            for t in th:
                t.join()
            return max(a.elapsed_time(b) for a, b in ev), sum(fl.stats()["launches"] for fl in flows)

        return {c: one for c in CALLS}, lambda: [fl.group_error() for fl in flows], flows, dense
    except BaseException:
        for d in dense:
            d.close()
        for fl in flows:
            fl.close()
        raise


def run(devs, s, reps, warmup):
    import torch
    rng = np.random.default_rng(1)
    x = None
    t = {}
    with skb.MultiFlow(devs) as mf:
        geometry(mf, s)
        operators(mf, s, 0, s["n_fib"], lambda nb, w, ex, ey, ez, ai: mf.set_body_operators([nb], w, ex, ey, ez, ai),
                  mf.set_fiber_links)
        mf.set_dense(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, s["M"])
        mf.set_dense(skb.DENSE_M_INV, s["M"])
        x = rng.normal(size=mf.solution_size())
        p = params(s, s["n_fib"])
        mcall = {"matvec": lambda: mf.apply_system_matvec(x, ETA),
                 "precondition": lambda: mf.apply_system_preconditioner(x),
                 "rhs": lambda: mf.build_system_rhs(*p, DT, ETA)}
        grp, errors, flows, dense = run_group(devs, s, x, reps, warmup)
        try:
            with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
                geometry(fl, s)
                operators(fl, s, 0, s["n_fib"],
                          lambda nb, w, ex, ey, ez, ai: fl.set_body_operators([nb], w, ex, ey, ez, ai),
                          fl.set_fiber_links)
                dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, s["M"])
                dn.set_matrix(skb.DENSE_M_INV, s["M"])
                d_x = torch.from_numpy(x).to("cuda:0")
                d_y = torch.empty_like(d_x)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

                def single(call):
                    st = torch.cuda.current_stream().cuda_stream
                    e0.record()
                    if call == "matvec":
                        fl.apply_system_matvec_device(dn, d_x.data_ptr(), ETA, d_y.data_ptr(), st)
                    elif call == "precondition":
                        fl.apply_system_preconditioner_device(dn, d_x.data_ptr(), d_y.data_ptr(), st)
                    else:
                        fl.build_system_rhs_device(*p, DT, ETA, 0, 0, 0, d_y.data_ptr(), stream=st)
                    e1.record()
                    torch.cuda.synchronize()
                    return e0.elapsed_time(e1), fl.stats()["launches"]

                def mflow(call):
                    mcall[call]()
                    st = mf.stats()
                    return st["device_ms"], st["launches"]

                forms = {"group": lambda c: grp[c](c), "mflow": mflow, "single": single}
                for c in CALLS:
                    for _ in range(warmup):
                        for f in forms.values():
                            f(c)
                    ts = {k: [] for k in forms}
                    for _ in range(reps):  # alternating, one call of each form per round
                        for k, f in forms.items():
                            ts[k].append(f(c))
                    t[c] = {k: summary(v) for k, v in ts.items()}
            t["group_error"] = errors()
        finally:
            for d in dense:
                d.close()
            for f in flows:
                f.close()
    return dict(devices=devs, calls=t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--devices", nargs="*", default=None, help="device lists, e.g. 0,0 0,1")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if capi.device_count() == 0:
        raise SystemExit("bench_group_system.py needs a GPU")
    if a.devices:
        lists = [[int(d) for d in v.split(",")] for v in a.devices]
    else:
        lists = [[0, 0]] + [list(range(k)) for k in (2, 4, 8) if capi.device_count() >= k]
    s = c3_shape(np.random.default_rng(0))
    s["Ainv_b"] = np.eye(3 * s["nbn"] + 6)
    out = dict(card=card(), case="C3 + 1 body x 400 nodes, 200 bound fibers",
               runs=[run(d, s, a.reps, a.warmup) for d in lists])
    print(json.dumps(out, indent=1))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

"""GPU test of the one-device flow's host-array calls interleaved on one flow.  Each call stages its inputs and outputs
in slots the flow owns, apart from the workspace the device cores read and write, so no call may see another call's
staged data as its own workspace, or the reverse, whatever the order of the calls, the sizes the slots were grown to
before, or the CUDA graphs the small matvec / velocity_at_targets replay in between.

Over rounds whose fiber count and target count grow and then shrink, every host-array call (skb_flow_fibers,
_periphery, _bodies, _velocity_at_targets, _matvec, _apply_matvec, _apply_matvec_dense, _build_fiber_rhs,
_apply_fiber_preconditioner, _apply_fiber_force, _fiber_matvec, _apply_system_matvec, _apply_system_preconditioner,
_build_system_rhs), optional inputs given and NULL, runs on one flow in an order that changes every round.  Each
result must be bitwise that of the same call on a flow set up fresh for the round, and that of its _device twin where
one exists."""
import contextlib

import numpy as np
import pytest

import skellysim_b200 as skb
from test_gpu_system_edges import ETA, DT, edge_case
from test_gpu_system_matvec import setup_flow

pytestmark = pytest.mark.gpu

SHAPE = dict(n_shell=300, n_body_nodes=600, n_bodies=2, nodes=(8, 16, 32))
ROUNDS = [(6, 5), (24, 700), (3, 2)]  # (fibers, targets): grown, then shrunk


def round_inputs(case, n_trg, seed):
    fib, shell, bodies, ops, links, x, params, fparams, src = case
    rng = np.random.default_rng(seed)
    nf, ns, nb, nfib = fib["pos"].shape[0], shell["pos"].shape[0], bodies["pos"].shape[0], len(fib["n_nodes"])
    return dict(r_trg=rng.uniform(-2, 2, (n_trg, 3)), r_small=rng.uniform(-2, 2, (2, 3)), ff=rng.normal(size=(nf, 3)),
                sd=rng.normal(size=(ns, 3)), bd=rng.normal(size=(nb, 3)), ft=src["ft"], x4=rng.normal(size=4 * nf),
                v=rng.normal(size=(nf, 3)), link=rng.normal(size=(nfib, 7)), f_ext=src["f_ext"], x=x, params=params,
                kw=dict(v_growth=src["v_growth"], force_scale=src["force_scale"]))


def set_up(fl, dn, case):
    fib, shell, bodies, ops, links, x, params, fparams, src = case
    setup_flow(fl, dn, fib, shell, bodies, ops, links)
    fl.set_point_sources(*src["points"])
    fl.set_background(*src["background"])


def host_calls(fl, dn, a):
    """name -> the host-array call on fl (optional inputs given and NULL)"""
    p, kw = a["params"], a["kw"]
    return {
        "fibers": lambda: fl.fiber_flow(a["r_trg"], a["ff"], ETA, subtract_self=False),
        "periphery": lambda: fl.periphery_flow(a["r_trg"], a["sd"], ETA),
        "bodies": lambda: fl.body_flow(a["r_trg"], a["bd"], a["ft"], ETA),
        "velocity_at_targets": lambda: fl.velocity_at_targets(a["r_trg"], a["ff"], a["sd"], a["bd"], a["ft"], ETA),
        "matvec": lambda: fl.matvec(a["ff"], a["sd"], a["bd"], a["ft"], ETA),
        "apply_matvec": lambda: fl.apply_matvec(a["x4"], a["sd"], a["bd"], a["ft"], ETA, a["link"]),
        "apply_matvec_unlinked": lambda: fl.apply_matvec(a["x4"], a["sd"], a["bd"], a["ft"], ETA),
        "apply_matvec_dense": lambda: fl.apply_matvec(a["x4"], a["sd"], a["bd"], a["ft"], ETA, a["link"], dense=dn),
        "build_fiber_rhs": lambda: fl.build_fiber_rhs(*p, DT, ETA, v_on_fibers=a["v"], f_external=a["f_ext"], **kw),
        "build_fiber_rhs_bare": lambda: fl.build_fiber_rhs(*p, DT, ETA),
        "apply_fiber_preconditioner": lambda: fl.apply_fiber_preconditioner(a["x4"]),
        "apply_fiber_force": lambda: fl.apply_fiber_force(a["x4"]),
        "fiber_matvec": lambda: fl.fiber_matvec(a["x4"], a["v"], a["link"]),
        "fiber_matvec_free": lambda: fl.fiber_matvec(a["x4"], a["v"]),
        "apply_system_matvec": lambda: fl.apply_system_matvec(a["x"], ETA, dense=dn),
        "apply_system_preconditioner": lambda: fl.apply_system_preconditioner(a["x"], dense=dn),
        "build_system_rhs": lambda: fl.build_system_rhs(*p, DT, ETA, f_external=a["f_ext"],
                                                        body_forces_torques=a["ft"], **kw),
        "build_system_rhs_unforced": lambda: fl.build_system_rhs(*p, DT, ETA, **kw),
    }


def small_calls(fl, a):
    """the small graphed calls: captured on their second identical call, replayed from the third"""
    return [fl.velocity_at_targets(a["r_small"], a["ff"], a["sd"], a["bd"], a["ft"], ETA) for _ in range(3)] + \
           [fl.matvec(a["ff"], a["sd"], a["bd"], a["ft"], ETA) for _ in range(3)]


def device_twins(fl, dn, a):
    """name -> the _device twin's result on fl, its outputs NaN first"""
    import torch
    dev = torch.device("cuda", 0)
    t = lambda v: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).reshape(-1).to(dev)
    nan = lambda n: torch.full((max(n, 1),), float("nan"), dtype=torch.float64, device=dev)
    p, kw = a["params"], a["kw"]
    nf, ns, nb, n = a["ff"].shape[0], a["sd"].shape[0], a["bd"].shape[0], a["x"].size
    d = {k: t(a[k]) for k in ("ff", "sd", "bd", "x4", "v", "link", "f_ext", "x")}
    F, T = t(a["ft"][:, :3]), t(a["ft"][:, 3:])
    o = {}

    def run(name, size, launch):
        out = nan(size)
        launch(out.data_ptr())
        torch.cuda.synchronize()
        o[name] = out[:size].cpu().numpy()

    run("matvec", 3 * (nf + ns + nb), lambda y: fl.matvec_device(d["ff"].data_ptr(), d["sd"].data_ptr(),
                                                                 d["bd"].data_ptr(), F.data_ptr(), T.data_ptr(), ETA, y))
    for name, dense, link in (("apply_matvec", None, d["link"]), ("apply_matvec_unlinked", None, None),
                              ("apply_matvec_dense", dn, d["link"])):
        res, v_s, v_b = nan(4 * nf), nan(3 * ns), nan(3 * nb)
        fl.apply_matvec_device(dense, d["x4"].data_ptr(), d["sd"].data_ptr(), d["bd"].data_ptr(), F.data_ptr(),
                               T.data_ptr(), link.data_ptr() if link is not None else 0, ETA, res.data_ptr(),
                               v_s.data_ptr(), v_b.data_ptr())
        torch.cuda.synchronize()
        o[name] = (res[:4 * nf].cpu().numpy(), v_s[:3 * ns].cpu().numpy(), v_b[:3 * nb].cpu().numpy())
    run("build_fiber_rhs", 4 * nf, lambda y: fl.build_fiber_rhs_device(*p, DT, ETA, d["v"].data_ptr(),
                                                                        d["f_ext"].data_ptr(), y, **kw))
    run("build_fiber_rhs_bare", 4 * nf, lambda y: fl.build_fiber_rhs_device(*p, DT, ETA, 0, 0, y))
    run("apply_fiber_preconditioner", 4 * nf, lambda y: fl.apply_fiber_preconditioner_device(d["x4"].data_ptr(), y))
    run("apply_fiber_force", 3 * nf, lambda y: fl.apply_fiber_force_device(d["x4"].data_ptr(), y))
    run("fiber_matvec", 4 * nf, lambda y: fl.fiber_matvec_device(d["x4"].data_ptr(), d["v"].data_ptr(),
                                                                  d["link"].data_ptr(), y))
    run("fiber_matvec_free", 4 * nf, lambda y: fl.fiber_matvec_device(d["x4"].data_ptr(), d["v"].data_ptr(), 0, y))
    run("apply_system_matvec", n, lambda y: fl.apply_system_matvec_device(dn, d["x"].data_ptr(), ETA, y))
    run("apply_system_preconditioner", n, lambda y: fl.apply_system_preconditioner_device(dn, d["x"].data_ptr(), y))
    run("build_system_rhs", n, lambda y: fl.build_system_rhs_device(*p, DT, ETA, d["f_ext"].data_ptr(), F.data_ptr(),
                                                                     T.data_ptr(), y, **kw))
    run("build_system_rhs_unforced", n, lambda y: fl.build_system_rhs_device(*p, DT, ETA, 0, 0, 0, y, **kw))
    return o


def flat(r):
    return np.concatenate([np.asarray(v).reshape(-1) for v in r]) if isinstance(r, tuple) else np.asarray(r).reshape(-1)


def same(got, ref):
    return flat(got).shape == flat(ref).shape and np.array_equal(flat(got), flat(ref))


@pytest.mark.parametrize("graphed", [False, True])
def test_interleaved_host_calls_match_a_fresh_flow_and_their_device_twins(graphed):
    rng = np.random.default_rng(17)
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0]))
        for r, (n_fibers, n_trg) in enumerate(ROUNDS):
            case = edge_case(dict(SHAPE, n_fibers=n_fibers), 40 + r)
            a = round_inputs(case, n_trg, 60 + r)
            with skb.Flow(0) as fresh, skb.Dense(device_ids=[0]) as dn_fresh:
                set_up(fresh, dn_fresh, case)
                ref = {k: call() for k, call in host_calls(fresh, dn_fresh, a).items()}
                ref_small = small_calls(fresh, a)[0::3]
            set_up(fl, dn, case)
            calls = host_calls(fl, dn, a)
            for k in rng.permutation(list(calls)):
                if graphed:
                    small = small_calls(fl, a)
                    assert all(same(v, ref_small[0]) for v in small[:3]) and \
                        all(same(v, ref_small[1]) for v in small[3:]), (r, "small calls before", k)
                got = calls[k]()
                assert np.isfinite(flat(got)).all() and same(got, ref[k]), (r, k)
            # the host forms again, in reverse order, after the slots all have their size for this round
            for k in reversed(list(calls)):
                assert same(calls[k](), ref[k]), (r, k, "again")
            twins = device_twins(fl, dn, a)
            for k, v in twins.items():
                assert np.isfinite(flat(v)).all() and same(v, ref[k]), (r, k, "device twin")

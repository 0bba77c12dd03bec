"""GPU parity tests of the multi-GPU flow layer: group members exchanging strengths and partial velocities through peer
memory (group_kernels.cuh) and skb_mflow, ONE process driving n devices (include/skelly_b200_flow.h).

On a 1-GPU box the exchange protocol is still exercised: a device may be listed twice, which gives two group members
(two windows, two streams, flag barriers, push / pull kernels) on the same GPU.  With >= 2 GPUs the same tests run over
NVLink.  Reference: the oracle's restatement of System::apply_matvec (system.cpp:269-324).  Tolerance 1e-12."""
import numpy as np
import pytest

import oracle as orc
import skellysim_b200 as skb
from conftest import rel_l2, rel_max
from skellysim_b200 import capi
from test_gpu_fiberops import load_ops, make_ops
from test_gpu_flow import ft_of, load, make_system

pytestmark = pytest.mark.gpu
TOL = 1e-12


def _check(u, ref, tol=TOL):
    assert np.isfinite(u).all()
    assert rel_max(u, ref) < tol, rel_max(u, ref)
    assert rel_l2(u, ref) < tol, rel_l2(u, ref)


def device_lists():
    """Member -> device maps to test: always two and three members on GPU 0; real multi-GPU lists when present."""
    n = capi.device_count()
    out = [[0], [0, 0], [0, 0, 0]]
    for k in (2, 4, 8):
        if n >= k:
            out.append(list(range(k)))
    return out


def load_m(mf, fib, shell, body):
    mf.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
    mf.set_periphery(shell["pos"], shell["normals"])
    mf.set_bodies(body["pos"], body["normals"], body["centers"])


# 40 fibers: below the symmetric kernel's threshold (own rows, plain kernel); 120 x (16..96): symmetric block rows + pull
@pytest.mark.parametrize("n_fibers,nodes", [(40, (8, 16, 24, 32)), (120, (16, 32, 48, 64, 96))])
def test_mflow_matvec_matches_oracle(n_fibers, nodes):
    fib, shell, body = make_system(100 + n_fibers, n_fibers, 700, 360, 3, nodes=nodes)
    eta = 1.3
    ref = orc.matvec_flow(fib, shell, body, eta)
    for devs in device_lists():
        with skb.MultiFlow(devs) as mf:
            load_m(mf, fib, shell, body)
            v = mf.matvec(fib["forces"], shell["density"], body["density"], ft_of(body), eta)
            v2 = mf.matvec(fib["forces"], shell["density"], body["density"], ft_of(body), eta)
            # strengths change, positions stay (GMRES iterations): the double-buffered windows alternate
            v3 = mf.matvec(2.0 * fib["forces"], 2.0 * shell["density"], 2.0 * body["density"], 2.0 * ft_of(body), eta)
            parts = [mf.partition(g) for g in range(len(devs))]
        _check(v, ref)
        assert np.array_equal(v, v2), f"not reproducible on devices {devs}"
        _check(v3, 2.0 * ref)
        # the partition covers every fiber / row exactly once
        assert parts[0][0] == 0 and parts[-1][1] == n_fibers
        for a, b in zip(parts, parts[1:]):
            assert a[1] == b[0] and a[3] == b[2] and a[5] == b[4]


def test_mflow_matvec_with_cross_kernel():
    # own fibers x ALL periphery nodes in one pass per member; the members' partial Stokeslet sums at the periphery rows are
    # pulled together like the fiber rows' partials
    fib, shell, body = make_system(9, 120, 600, 200, 2, nodes=(16, 32, 48, 64, 96))
    eta = 1.4
    ref = orc.matvec_flow(fib, shell, body, eta)
    for devs in device_lists():
        with skb.MultiFlow(devs) as mf:
            load_m(mf, fib, shell, body)
            mf.set_cross(1)
            v = mf.matvec(fib["forces"], shell["density"], body["density"], ft_of(body), eta)
            v2 = mf.matvec(fib["forces"], shell["density"], body["density"], ft_of(body), eta)
        _check(v, ref)
        assert np.array_equal(v, v2)


def test_mflow_matvec_with_fused_self_exclusion():
    fib, shell, body = make_system(7, 120, 500, 200, 2, nodes=(16, 32, 48, 64, 96))
    eta = 0.8
    ref = orc.matvec_flow(fib, shell, body, eta)
    for devs in ([0, 0], [0, 0, 0]):
        for cross in (0, 1):
            with skb.MultiFlow(devs) as mf:
                load_m(mf, fib, shell, body)
                mf.set_cross(cross)
                mf.set_self_exclusion(True)
                print("exclusion: devices", devs, "cross", cross, flush=True)
                v = mf.matvec(fib["forces"], shell["density"], body["density"], ft_of(body), eta)
            _check(v, ref)


@pytest.mark.parametrize("with_dense", [False, True])
def test_mflow_apply_matvec_matches_oracle(with_dense):
    fib, shell, body = make_system(31, 110, 400, 240, 2, nodes=(16, 24, 32, 48, 64))
    ops = make_ops(fib, 5)
    rng = np.random.default_rng(9)
    nf, ns = fib["pos"].shape[0], shell["pos"].shape[0]
    x = rng.normal(size=4 * nf)
    link = rng.normal(size=(len(fib["n_nodes"]), 7))
    eta = 1.1
    res_ref, v_ref = orc.apply_matvec_fibers(fib, shell, body, ops, x, eta, link)
    v_shell_ref, v_body_ref = v_ref[nf:nf + ns], v_ref[nf + ns:]
    A = rng.normal(size=(3 * ns, 3 * ns)) / np.sqrt(3 * ns) if with_dense else None
    shell_ref = v_shell_ref if A is None else (A @ shell["density"].reshape(-1)).reshape(-1, 3) + v_shell_ref
    for devs in device_lists():
        with skb.MultiFlow(devs) as mf:
            load_m(mf, fib, shell, body)
            for n in ops["D_1_0"]:
                mf.set_fiber_class(n, ops["D_1_0"][n], ops["P"][n])
            mf.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
            if A is not None:
                mf.set_dense(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, A)
            res, out_s, v_b = mf.apply_matvec(x, shell["density"], body["density"], ft_of(body), eta, link)
            st = mf.stats()
        _check(res, res_ref)
        _check(out_s, shell_ref)
        _check(v_b, v_body_ref)
        assert st["launches"] > 0 and st["n_pairs"] > 0


def test_resized_geometry_matches_a_fresh_multiflow():
    """Grow the fibers, then the periphery, then the bodies of one MultiFlow, and shrink them again in reverse order.
    After every change each host-array call (matvec, apply_matvec with and without the periphery's dense operator, the
    whole-system matvec, preconditioner and RHS) gives bitwise what a MultiFlow set up directly on that geometry gives:
    every call stages its members' transfers for the sizes it meets, also for members that share a device."""
    from test_gpu_system_edges import DT, ETA, edge_case, partial_inputs, setup_mflow_edges

    small = dict(n_fibers=24, nodes=(8, 16), n_shell=200, n_body_nodes=400, n_bodies=2)
    grown = [dict(small, n_fibers=40)]
    grown.append(dict(grown[-1], n_shell=300))
    grown.append(dict(grown[-1], n_body_nodes=600, n_bodies=3))
    shapes = [small] + grown + grown[-2::-1] + [small]
    cases = [edge_case(kw, 60 + i) for i, kw in enumerate(shapes)]

    def set_up(mf, case, dense):
        fib, shell, bodies, ops, links = case[:5]
        if dense:
            setup_mflow_edges(mf, fib, shell, bodies, ops, links)
            return
        load_m(mf, fib, shell, bodies)
        for n in ops["D_1_0"]:
            mf.set_fiber_class(n, ops["D_1_0"][n], ops["P"][n])
        mf.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])

    def calls(mf, case, dense):
        fib, shell, bodies, ops, links, x, params, _, src = case
        strengths, partial, _ = partial_inputs(fib, shell, bodies, x, 70)
        link = np.random.default_rng(71).normal(size=(len(fib["n_nodes"]), 7))
        if dense:
            mf.set_point_sources(*src["points"])
            mf.set_background(*src["background"])
        out = [mf.matvec(*strengths, ETA), *mf.apply_matvec(*partial, ETA, link)]
        if dense:
            out += [mf.apply_system_matvec(x, ETA), mf.apply_system_preconditioner(x),
                    mf.build_system_rhs(*params, DT, ETA, f_external=src["f_ext"], body_forces_torques=src["ft"],
                                        v_growth=src["v_growth"], force_scale=src["force_scale"])]
        return out

    for devs in device_lists()[1:]:
        for dense in (False, True):
            with skb.MultiFlow(devs) as mf:
                for kw, case in zip(shapes, cases):
                    set_up(mf, case, dense)
                    got = calls(mf, case, dense)
                    with skb.MultiFlow(devs) as fresh:
                        set_up(fresh, case, dense)
                        want = calls(fresh, case, dense)
                    assert len(got) == (7 if dense else 4)
                    for k, (g, w) in enumerate(zip(got, want)):
                        assert np.array_equal(g, w), (devs, dense, kw, k)


def test_mflow_velocity_at_targets():
    fib, shell, body = make_system(77, 30, 300, 120, 1)
    rng = np.random.default_rng(3)
    r_trg = rng.uniform(-3, 3, (1001, 3))
    eta = 0.9
    ref = (orc.fiber_flow(r_trg, fib["pos"], fib["n_nodes"], fib["lengths"], fib["forces"], eta, subtract_self=False)
           + orc.body_flow(r_trg, body["pos"], body["normals"], body["density"], body["centers"], body["forces"],
                           body["torques"], eta)
           + orc.periphery_flow(r_trg, shell["pos"], shell["normals"], shell["density"], eta))
    for devs in device_lists():
        with skb.MultiFlow(devs) as mf:
            load_m(mf, fib, shell, body)
            v = mf.velocity_at_targets(r_trg, fib["forces"], shell["density"], body["density"], ft_of(body), eta)
        _check(v, ref)


def test_group_members_in_one_process_by_hand():
    # what skb_mflow does internally, spelled out with the group calls a rank-per-GPU host uses (connect instead of
    # export / import because both members live in this process)
    fib, shell, body = make_system(5, 100, 300, 100, 1, nodes=(32, 48))
    nfib = len(fib["n_nodes"])
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
    ns, nb, nf = shell["pos"].shape[0], body["pos"].shape[0], fib["pos"].shape[0]
    eta = 1.0
    ref = orc.matvec_flow(fib, shell, body, eta)
    cut_f, cut_s, cut_b = nfib // 2, ns // 3, nb // 2
    ranges = [(0, cut_f, 0, cut_s, 0, cut_b), (cut_f, nfib, cut_s, ns, cut_b, nb)]
    import torch
    members = [skb.Flow(0), skb.Flow(0)]
    try:
        for g, fl in enumerate(members):
            load(fl, fib, shell, body)
            fl.set_target_ranges(*ranges[g])
            fl.group_init(g, 2)
        members[0].group_connect(1, members[1])
        members[1].group_connect(0, members[0])
        for fl in members:   # members share GPU 0: all allocations before the first flag wait
            fl.group_warmup()
        outs, streams = [], [torch.cuda.Stream(), torch.cuda.Stream()]
        dev = torch.device("cuda", 0)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        for g, fl in enumerate(members):
            f0, f1, s0, s1, b0, b1 = ranges[g]
            ins = [t(fib["forces"][off[f0]:off[f1]]), t(shell["density"][s0:s1]), t(body["density"]), t(body["forces"]),
                   t(body["torques"])]
            out = torch.empty(((off[f1] - off[f0]) + (s1 - s0) + (b1 - b0), 3), dtype=torch.float64, device=dev)
            outs.append((out, ins))
        torch.cuda.synchronize()
        # (no host synchronisation between the two launches: member 0 sits in its flag wait until member 1 has pushed)
        for g, fl in enumerate(members):
            out, ins = outs[g]
            fl.matvec_device(*[x.data_ptr() for x in ins], eta, out.data_ptr(), streams[g].cuda_stream)
        torch.cuda.synchronize()
        assert all(fl.group_error() < 0 for fl in members)
        for g in range(2):
            f0, f1, s0, s1, b0, b1 = ranges[g]
            want = np.concatenate([ref[off[f0]:off[f1]], ref[nf + s0:nf + s1], ref[nf + ns + b0:nf + ns + b1]])
            _check(outs[g][0].cpu().numpy(), want)
    finally:
        for fl in members:
            fl.close()

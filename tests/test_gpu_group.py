"""GPU tests of a group member's refusals, solo mode and leaving a group (skb_flow_group_*, include/skelly_b200_flow.h).

Both members of a group live on GPU 0 in this process.  No case here reaches a flag wait: the exchange itself (push,
flags, pull with two and three members) is covered by test_gpu_mflow.py."""
import numpy as np
import pytest

import oracle as orc
import skellysim_b200 as skb
from conftest import rel_l2, rel_max
from skellysim_b200 import capi
from test_gpu_flow import ft_of, load, make_system

pytestmark = pytest.mark.gpu
TOL = 1e-12
SKB_ERR_INVALID, SKB_ERR_STATE = 1, 4


def _system(n_fibers=120, nodes=(16, 32, 48, 64, 96), seed=220):
    # 120 fibers of 16..96 nodes: enough for the symmetric block rows of a 2-group (partial sums + pull)
    return make_system(seed, n_fibers, 700, 360, 3, nodes=nodes)


def _halves(fib, shell, body):
    nfib, ns, nb = len(fib["n_nodes"]), shell["pos"].shape[0], body["pos"].shape[0]
    return [(0, nfib // 2, 0, ns // 3, 0, nb // 2), (nfib // 2, nfib, ns // 3, ns, nb // 2, nb)]


def _refused(code, text, call):
    with pytest.raises(capi.SkbError, match=f"error {code}: .*{text}"):
        call()


def _member(fib, shell, body, rank, size, ranges):
    fl = skb.Flow(0)
    load(fl, fib, shell, body)
    fl.set_target_ranges(*ranges)
    fl.group_init(rank, size)
    return fl


def _matvec(fl, fib, shell, body, eta=1.3):
    return fl.matvec(fib["forces"], shell["density"], body["density"], ft_of(body), eta)


def test_matvec_with_a_missing_peer_is_refused():
    fib, shell, body = _system()
    fl = _member(fib, shell, body, 0, 2, _halves(fib, shell, body)[0])
    try:
        fl.group_warmup()  # alone: no flags, own window only
        before = capi.launch_count()
        _refused(SKB_ERR_STATE, "not all peers are connected", lambda: _matvec(fl, fib, shell, body))
        assert capi.launch_count() == before
    finally:
        fl.close()


def test_matvec_after_the_geometry_was_resized_is_refused():
    fib, shell, body = _system()
    fl = _member(fib, shell, body, 0, 2, _halves(fib, shell, body)[0])
    try:
        fib2 = _system(n_fibers=100)[0]
        assert fib2["pos"].shape[0] != fib["pos"].shape[0]
        fl.set_fibers(fib2["pos"], fib2["n_nodes"], fib2["lengths"])
        before = capi.launch_count()
        _refused(SKB_ERR_STATE, "re-initialise the group", lambda: _matvec(fl, fib2, shell, body))
        assert capi.launch_count() == before
    finally:
        fl.close()


def test_connect_export_and_import_checks():
    fib, shell, body = _system()
    halves = _halves(fib, shell, body)
    fib2 = _system(n_fibers=100)[0]
    a = _member(fib, shell, body, 0, 2, halves[0])
    b = _member(fib2, shell, body, 1, 2, (50, 100, 0, 1, 0, 1))  # laid out for other fibers
    c = _member(fib, shell, body, 1, 2, halves[1])
    plain = skb.Flow(0)  # never in a group
    single = skb.Flow(0)
    try:
        load(plain, fib, shell, body)
        load(single, fib, shell, body)
        single.group_init(0, 1)  # leaves it a plain flow
        _refused(SKB_ERR_INVALID, "different geometries", lambda: a.group_connect(1, b))
        _refused(SKB_ERR_INVALID, "bad arguments", lambda: a.group_connect(0, c))  # own rank; c is rank 1
        _refused(SKB_ERR_INVALID, "bad arguments", lambda: a.group_connect(2, c))  # beyond the group
        for fl in (plain, single):
            _refused(SKB_ERR_INVALID, "no group window", fl.group_export)
            _refused(SKB_ERR_INVALID, "bad arguments", lambda: fl.group_import(1, bytes(64)))
            _refused(SKB_ERR_INVALID, "bad arguments", lambda: fl.group_connect(1, c))
            _refused(SKB_ERR_INVALID, "bad arguments", lambda: c.group_connect(0, fl))
        a.group_connect(1, c)  # the checks refuse nothing a matching pair needs
    finally:
        for fl in (a, b, c, plain, single):
            fl.close()


def test_solo_member_completes_matvec_device():
    import torch
    fib, shell, body = _system()
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
    f0, f1, s0, s1, b0, b1 = ranges = _halves(fib, shell, body)[1]
    fl = _member(fib, shell, body, 1, 2, ranges)
    try:
        fl.group_warmup()
        fl.group_set_solo(True)  # scripts/rank_share.py: this member's share alone
        dev = torch.device("cuda", 0)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        ins = [t(fib["forces"][off[f0]:off[f1]]), t(shell["density"][s0:s1]), t(body["density"]), t(body["forces"]),
               t(body["torques"])]
        outs = []
        for _ in range(2):
            out = torch.full(((off[f1] - off[f0]) + (s1 - s0) + (b1 - b0), 3), np.nan, dtype=torch.float64,
                             device=dev)
            fl.matvec_device(*[x.data_ptr() for x in ins], 1.3, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
            outs.append(out)
        torch.cuda.synchronize()
        u, u2 = (o.cpu().numpy() for o in outs)
        assert np.isfinite(u).all()
        assert np.array_equal(u, u2)
        assert fl.group_error() == -1
    finally:
        fl.close()


def test_leaving_a_group_restores_a_plain_flow():
    fib, shell, body = _system()
    nfib, ns, nb = len(fib["n_nodes"]), shell["pos"].shape[0], body["pos"].shape[0]
    eta = 1.3
    fl = _member(fib, shell, body, 0, 2, _halves(fib, shell, body)[0])
    try:
        fl.group_warmup()
        fl.group_init(0, 1)
        _refused(SKB_ERR_INVALID, "not a group member", lambda: fl.group_set_solo(True))
        assert fl.group_error() == -1
        fl.set_target_ranges(0, nfib, 0, ns, 0, nb)
        u = _matvec(fl, fib, shell, body, eta)
    finally:
        fl.close()
    ref = orc.matvec_flow(fib, shell, body, eta)
    assert np.isfinite(u).all()
    assert rel_max(u, ref) < TOL, rel_max(u, ref)
    assert rel_l2(u, ref) < TOL, rel_l2(u, ref)

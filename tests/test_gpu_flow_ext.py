"""The flows at targets and the matvec's v_all held row by row to the long-double restatement of tests/flow_reference.py:
|dev - ext| <= K u S per row component, K fixed from the kernel source before any GPU run (the module's docstring derives
it).  A normwise gate is set by the largest row; this one also holds the fiber rows, where the pair sum and the
subtracted self term cancel, the small kernels (the self term, the point sources' Oseen and rotlet kernels, the
background), the eps boundaries of their regularised branches, and the order in which the parts are composed.  Small
systems check every row; large ones the rows of pair_sum_reference.sample_rows.

The fused self-exclusion (set_self_exclusion(True)) skips every intra-fiber pair, so at the pairs within EPS it does not
reproduce the reference's non-cancelling rows; the matvec test asserts that it misses the bound there and meets it
everywhere else.

Worst ratio / K per quantity (test_worst_ratios_report prints them), on an H100 80GB HBM3 at 700 W:
    fiber_flow without / with the self term (2 .. 1100 nodes, eps edges)       0.00627 / 0.00625
    fiber_flow, one fiber of 4266 nodes (symmetric kernel)                     0.00333
    periphery_flow / body_flow                                                 0.0107 / 0.0189
    velocity_at_targets / velocity_field free rows                             0.00462 / 0.00955
    matvec plain / windows with f0 > 0                                         0.00577 / 0.00577
    matvec fast path, cross -1 / cross 0                                       0.00162 / 0.00162
    MultiFlow matvec, plain members / symmetric partials and pull              0.0121 / 0.00155
A self term whose j loop stops at n - 1, or that regularises at r < EPS, fails test_fiber_flow_every_row and
test_matvec_every_row_and_windows_that_tile_it.
"""
import numpy as np
import pytest

import flow_reference as fr
import pair_sum_reference as ps
import skellysim_b200 as skb
from skellysim_b200 import capi
from test_flow_ext_cpu import BG, edge_fibers, edge_targets, point_sources, shell_and_bodies
from test_gpu_flow import ft_of, load

pytestmark = pytest.mark.gpu
WORST = {}
SIZES = (2, 3, 4, 7, 8, 31, 32, 33, 64, 127, 128, 129, 1100)


def _check(name, dev, ref, rows=None):
    """every component of every row within its K; records the worst ratio / K under `name`"""
    ext, S, K = ref
    dev = np.asarray(dev)
    if rows is not None:
        dev = dev[rows]
    assert np.isfinite(dev).all(), name
    r = fr.ratio(dev, ext, S) / np.asarray(K, dtype=np.float64)[:, None]
    w = float(r.max()) if r.size else 0.0
    WORST[name] = max(WORST.get(name, 0.0), w)
    bad = np.argwhere(r > 1)
    assert bad.size == 0, (name, bad[:5].tolist(), w)


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _k_sym(n_src, n_trg, rows, n_parts=1):
    """the symmetric kernel's K at the leading rows (every part of an n_parts partition, plus the pull's adds)"""
    rows = np.asarray(rows)
    rows = rows[rows < n_src]
    if n_src < 2 * ps.SYM_BLOCK or rows.size == 0:
        return 0
    nb = ps.n_pad(n_src) // ps.SYM_BLOCK
    return max(float(ps.k_sym_rows(n_src, n_trg, rows, p, n_parts,
                                   plan=capi.sym_plan_query(nb, p, n_parts, num_sms=_num_sms())).max())
               for p in range(n_parts)) + (n_parts if n_parts > 1 else 0)


def _system(seed, nodes=SIZES, n_shell=300, per=40, subnormal=True):
    rng = np.random.default_rng(seed)
    fib = edge_fibers(rng, nodes)
    if subnormal:   # one fiber's nodes 1e-160 apart: r^2 subnormal, masked by the pair kernel, subtracted by the self term
        x = np.array([[0.0, 2.7, 2.7], [1e-160, 2.7, 2.7], [0.5, 2.7, 2.7]])
        fib = dict(pos=np.concatenate([fib["pos"], x]), n_nodes=fib["n_nodes"] + [3],
                   lengths=fib["lengths"] + [0.5], forces=np.concatenate([fib["forces"], rng.normal(size=(3, 3))]))
    shell, body = shell_and_bodies(rng, n_shell, per)
    return rng, fib, shell, body


def _flow(fib, shell, body, points=None, bg=None):
    fl = skb.Flow(0)
    load(fl, fib, shell, body)
    if points is not None:
        fl.set_point_sources(*points)
    if bg is not None:
        fl.set_background(*bg)
    return fl


# ---- fiber flow ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("eta", [0.37, 2.5])
def test_fiber_flow_every_row(eta):
    rng, fib, shell, body = _system(1)
    r = np.concatenate([fib["pos"], rng.uniform(-3, 3, (300, 3)), fib["pos"][:40] + 1e-7])
    with _flow(fib, shell, body) as fl:
        v = fl.fiber_flow(r, fib["forces"], eta, subtract_self=False)
        vs = fl.fiber_flow(r, fib["forces"], eta, subtract_self=True)
        assert np.array_equal(vs, fl.fiber_flow(r, fib["forces"], eta, subtract_self=True))
    _check("fiber_flow", v, fr.fiber_flow(fib, r, eta))
    _check("fiber_flow subtract_self", vs, fr.fiber_flow(fib, r, eta, True))


def test_largest_fiber_and_its_refusal():
    """4266 nodes (48 B/node of shared memory: 199.97 KB, within the 200 KB set_fibers allows) runs with the self term;
    4267 is refused and leaves the flow as it was"""
    rng = np.random.default_rng(2)
    n = 4266
    h = rng.normal(size=3)
    pos = np.linspace(0, 3.0, n)[:, None] * (h / np.linalg.norm(h)) + rng.uniform(-1, 1, 3)
    pos[1] = pos[0] + [fr.EPS, 0, 0]          # two nodes exactly EPS apart along x
    fib = dict(pos=np.concatenate([pos, pos[:7] + 0.5]), n_nodes=[n, 7], lengths=[3.0, 0.02],
               forces=rng.normal(size=(n + 7, 3)) * 10.0 ** rng.uniform(-3, 3, (n + 7, 1)))
    r = np.concatenate([fib["pos"], rng.uniform(-2, 2, (200, 3))])
    rows = ps.sample_rows(len(r), (128, ps.SYM_BLOCK), n_lead=len(fib["pos"]), full_limit=0)
    rows = np.unique(np.concatenate([rows, np.arange(8)]))
    big = dict(pos=np.concatenate([pos, [[9.0, 9, 9]], pos[:7] + 0.5]), n_nodes=[n + 1, 7])
    eta = 0.37
    with skb.Flow(0) as fl:
        fl.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
        v = fl.fiber_flow(r, fib["forces"], eta, subtract_self=True)
        with pytest.raises(RuntimeError):
            fl.set_fibers(big["pos"], big["n_nodes"], fib["lengths"])
        assert np.array_equal(v, fl.fiber_flow(r, fib["forces"], eta, subtract_self=True))
        fl.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
        assert np.array_equal(v, fl.fiber_flow(r, fib["forces"], eta, subtract_self=True))
    ref = fr.fiber_flow(fib, r[rows], eta, True, k=_k_sym(len(fib["pos"]), len(r), rows),
                        nodes=np.where(rows < len(fib["pos"]), rows, -1))
    _check("fiber_flow 4266 nodes", v, ref, rows)


# ---- the other classes and the sum at targets ---------------------------------------------------------------------
@pytest.mark.parametrize("eta", [0.37, 2.5])
def test_periphery_and_body_flows_every_row(eta):
    rng, fib, shell, body = _system(3, nodes=(8, 16))
    r = np.concatenate([rng.uniform(-3, 3, (400, 3)), body["centers"], body["pos"],
                        body["centers"][0] + [[fr.EPS, 0, 0], [np.nextafter(fr.EPS, 0), 0, 0]]])
    ft = ft_of(body)
    with _flow(fib, shell, body) as fl:
        vs = fl.periphery_flow(r, shell["density"], eta)
        vb = fl.body_flow(r, body["density"], ft, eta)
    _check("periphery_flow", vs, fr.compose(fr.periphery_flow(shell, r, eta)))
    _check("body_flow", vb, fr.compose(*fr.body_flow(body, r, eta)))


@pytest.mark.parametrize("eta", [0.37, 2.5])
def test_velocity_at_targets_every_row(eta):
    rng, fib, shell, body = _system(4)
    points = point_sources(rng)
    r = edge_targets(rng, fib, body, points[0], n_free=500)
    with _flow(fib, shell, body, points, BG) as fl:
        v = fl.velocity_at_targets(r, fib["forces"], shell["density"], body["density"], ft_of(body), eta)
        v6 = fl.velocity_at_targets(r[-6:], fib["forces"], shell["density"], body["density"], ft_of(body), eta)
    ref = fr.velocity_at_targets(fib, shell, body, r, eta, points, BG)
    _check("velocity_at_targets", v, ref)
    _check("velocity_at_targets", v6, fr.take(ref, slice(len(r) - 6, None)))


def test_velocity_field_free_rows_bound_interior_rows_bitwise():
    rng, fib, shell, body = _system(5, nodes=(8, 16, 33))
    points = point_sources(rng)
    kind, radii = np.array([1, 1, 2], dtype=np.int32), np.array([[0.4, 0, 0], [0.4, 0, 0], [0.5, 0.3, 0.35]])
    uw = rng.uniform(-0.5, 0.5, (3, 6))
    c = body["centers"]
    r = np.concatenate([rng.uniform(-2.5, 2.5, (400, 3)), c[1] + rng.uniform(-0.3, 0.3, (150, 3)),
                        c[2] + rng.uniform(-0.4, 0.4, (100, 3)), c[0] + rng.uniform(-0.3, 0.3, (50, 3))])
    eta = 0.37
    with _flow(fib, shell, body, points, BG) as fl:
        fl.set_listener_frame(fib["forces"], shell["density"], body["density"], ft_of(body), uw, kind, radii, eta)
        v = fl.velocity_field(r)
    ref, inside, rigid = fr.velocity_field(fib, shell, body, r, eta, kind, radii, uw, points, BG)
    both = fr.interior(r, dict(centers=c[1:2]), kind[1:2], radii[1:2], uw[1:2])[0] & \
        fr.interior(r, dict(centers=c[2:]), kind[2:], radii[2:], uw[2:])[0]
    assert both.sum() > 10 and (~inside).sum() > 300
    assert np.array_equal(v[inside], rigid[inside])          # the last matching body's U + omega x dx, bitwise
    _check("velocity_field free rows", v[~inside], fr.take(ref, ~inside))


# ---- the matvec's v_all -------------------------------------------------------------------------------------------
def _matvec(fl, fib, shell, body, eta):
    return fl.matvec(fib["forces"], shell["density"], body["density"], ft_of(body), eta)


@pytest.mark.parametrize("eta", [0.37, 2.5])
def test_matvec_every_row_and_windows_that_tile_it(eta):
    _, fib, shell, body = _system(6)
    nfib, ns, nb = len(fib["n_nodes"]), len(shell["pos"]), len(body["pos"])
    cuts = [(0, 3, 0, 50, 0, 30), (3, 11, 50, 51, 30, 90), (11, nfib, 51, ns, 90, nb)]
    with _flow(fib, shell, body) as fl:
        v = _matvec(fl, fib, shell, body, eta)
        parts = []
        for rg in cuts:
            fl.set_target_ranges(*rg)
            parts.append(_matvec(fl, fib, shell, body, eta))
        fl.set_target_ranges(0, nfib, 0, ns, 0, nb)
        fl.set_self_exclusion(True)
        v_excl = _matvec(fl, fib, shell, body, eta)
    ref = fr.matvec(fib, shell, body, eta)
    _check("matvec plain", v, ref)
    for rg, p in zip(cuts, parts):
        _check("matvec windows f0 > 0", p, fr.matvec(fib, shell, body, eta, rg))
    # the fused exclusion skips every intra-fiber pair, so within EPS it does not meet the reference's non-cancelling
    # rows (the unregularised pair minus the regularised one); elsewhere it agrees to rounding
    ext, S, K = ref
    r = fr.ratio(v_excl, ext, S) / K[:, None]
    nf = len(fib["pos"])
    near = np.zeros(len(v), dtype=bool)
    near[[0, 1, 9, 10, nf - 3, nf - 2]] = True   # r == EPS, 0 < r < EPS (edge_fibers) and the subnormal r^2 (_system)
    assert (r[near].max(axis=1) > 1e6).all() and r[~near].max() <= 1


def _fast_system(seed):
    """>= 4096 fiber nodes (the symmetric kernel) and >= 256 periphery nodes (the cross kernel)"""
    _, fib, shell, body = _system(seed, nodes=SIZES + (1100, 1100, 900))
    assert len(fib["pos"]) >= 4096 and len(shell["pos"]) >= 256
    return fib, shell, body


def _fast_rows(nf, n_all):
    rows = ps.sample_rows(n_all, (ps.SYM_BLOCK, ps.SYM_GROUP, ps.CROSS_BLOCK), n_lead=nf, ragged_period=ps.SYM_GROUP,
                          full_limit=0)
    return np.unique(np.concatenate([rows, np.arange(40), np.arange(nf, nf + 40), np.arange(n_all - 40, n_all)]))


@pytest.mark.parametrize("cross", [-1, 0])
def test_matvec_fast_path_rows(cross):
    fib, shell, body = _fast_system(7)
    nf, n_all = len(fib["pos"]), len(fib["pos"]) + len(shell["pos"]) + len(body["pos"])
    eta = 2.5
    rows = _fast_rows(nf, n_all)
    with _flow(fib, shell, body) as fl:
        fl.set_cross(cross)
        out = {}
        for ov in (True, False):
            fl.set_overlap(ov)
            out[ov] = _matvec(fl, fib, shell, body, eta)
    assert np.array_equal(out[True], out[False])
    _check(f"matvec fast path cross {cross}", out[True],
           fr.matvec(fib, shell, body, eta, k_fib=_k_sym(nf, n_all, rows), rows=rows), rows)


def _device_lists():
    return [[0, 0]] + ([[0, 1]] if capi.device_count() >= 2 else [])


@pytest.mark.parametrize("fast", [False, True])
def test_mflow_matvec_rows(fast):
    """skb_mflow's group members: the plain kernel on their own rows (small), or the symmetric kernel's partial rows
    pulled together, the self term subtracted after the pull (fast)"""
    if fast:
        fib, shell, body = _fast_system(8)
    else:
        _, fib, shell, body = _system(8, nodes=(8, 16, 31, 64, 127, 128, 129))
    nf, n_all = len(fib["pos"]), len(fib["pos"]) + len(shell["pos"]) + len(body["pos"])
    rows = _fast_rows(nf, n_all) if fast else np.arange(n_all)
    eta = 0.37
    for devs in _device_lists():
        with skb.MultiFlow(devs) as mf:
            load(mf, fib, shell, body)
            v = _matvec(mf, fib, shell, body, eta)
        k = _k_sym(nf, n_all, rows, n_parts=len(devs)) if fast else None
        _check(f"MultiFlow matvec {'fast' if fast else 'plain'}", v,
               fr.matvec(fib, shell, body, eta, k_fib=k, rows=rows), rows)


def test_worst_ratios_report():
    print("\nworst ratio / K:")
    for k, v in sorted(WORST.items()):
        print(f"    {k:42s} {v:.3g}")

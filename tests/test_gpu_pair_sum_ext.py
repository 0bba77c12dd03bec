"""Every sampled target row of the plain pair kernel (pair_sum_kernel), the symmetric kernel (pair_sym_kernel) and the
fiber-periphery cross kernel (pair_cross_kernel) held to the long-double restatement of tests/pair_sum_reference.py:
|dev - ext| <= K u S per row component, K fixed from each launch's plan before any GPU run (the module's docstring
derives it).  A normwise gate is set by the largest row; this one also sees the rows whose true value is small against
the terms summed into them: far targets, cancelling sources, the ragged last tile, one member's rows of a symmetric
partition and the periphery rows written by the cross kernel's reverse sums.  Small shapes check every row; large ones
the rows of pair_sum_reference.sample_rows (tile, block and group edges, the ragged last tile, the remainder targets
and 256 random rows).  Every call is repeated once and must be bitwise equal.

The symmetric kernel runs from two 1024-node blocks of sources on (below that the plain kernel serves the call), so its
shapes are 2048, 2049 (+ 300 remainder targets), 3071 and 4097 (+ 4097), and the partitions n_parts in {2, 3} at 4097.

Worst ratio / K per kernel and mode (test_worst_ratios_report prints them), on an H100 80GB HBM3 at 700 W.  The bounds
are worst-case counts, so every ratio is far below 1; a slip in the pair formula or the summation structure misses its
bound by 1e9 or more (tests/test_pair_sum_ext_cpu.py), a second-order rsqrt step by ~30x on the single-pair rows:
    plain sl / excl / dl9 / dl6 (every row, T in 1, 2, 4, 8, forced S)   0.106 / 0.106 / 0.0848 / 0.106
    plain sl / dl9 single pair                                           0.0883 / 0.0959
    plain sl / dl9 cancellation and wide range                           0.0623 / 0.0301
    plain sl / dl9 planner 3001 x 2500                                   0.00209 / 0.0113
    plain sl / dl9 1 x 32767 and 1 x 40001 (wide reduce)                 1.26e-4 / 9.87e-4
    symmetric / partition / duplicates / exclusion                      2.39e-4 / 1.62e-4 / 1.78e-4 / 1.79e-4
    cross periphery rows / fiber rows                                    2.64e-4 / 4.04e-3
    cross off: periphery rows / fiber rows                               1.67e-4 / 4.16e-3
"""
import numpy as np
import pytest

import pair_sum_reference as ps
import skellysim_b200 as skb
from skellysim_b200 import capi

pytestmark = pytest.mark.gpu
SL, DL = skb.KERNEL_STOKESLET, skb.KERNEL_STRESSLET
WORST = {}


def _check(name, dev, ext, S, K):
    """every component of every row within its K; records the worst ratio / K under `name`"""
    dev = np.asarray(dev)
    assert np.isfinite(dev).all(), name
    K = np.broadcast_to(np.asarray(K, dtype=np.float64).reshape(-1, 1) if np.ndim(K) else K, dev.shape)
    r = ps.ratio(dev, ext, S) / K
    w = float(r.max()) if r.size else 0.0
    WORST[name] = max(WORST.get(name, 0.0), w)
    bad = np.argwhere(r > 1)
    assert bad.size == 0, (name, bad[:5].tolist(), w)


def _num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _twice(fn):
    a, b = fn(), fn()
    assert np.array_equal(a, b), "bitwise reproducible"
    return a


def _plain_k(c, kind, n_trg, n_src, force_S=0):
    st = c.stats()
    p = capi.plan_query(SL if kind == "sl" else DL, n_trg, n_src, force_T=st["targets_per_thread"],
                        force_S=force_S or st["source_splits"])
    assert p["n_splits"] == st["source_splits"]
    return ps.k_plain(kind, n_src, p["tiles_per_split"], p["n_splits"]), p


# ---- plain kernel -------------------------------------------------------------------------------------------------
TUNINGS = [(1, 0), (2, 0), (4, 0), (8, 0), (2, 3), (8, 5), (0, 0)]


def _plain_geometry(seed, n_src, n_extra):
    rng = np.random.default_rng(seed)
    rs = rng.uniform(-1, 1, (n_src, 3))
    rt = np.concatenate([rs, rng.uniform(-1.2, 1.2, (n_extra, 3))])
    n_nodes = rng.choice([3, 8, 13], size=n_src)
    ids = np.repeat(np.arange(n_src), n_nodes)[:n_src].astype(np.int32)
    return rng, rs, rt, ids


@pytest.mark.parametrize("n_src,n_extra", [(1, 700), (2, 301), (127, 1), (128, 129), (129, 900), (333, 1037)])
def test_plain_kernel_every_row(n_src, n_extra):
    rng, rs, rt, ids = _plain_geometry(n_src, n_src, n_extra)
    n_trg = rt.shape[0]
    f, f9 = rng.normal(size=(n_src, 3)), rng.normal(size=(n_src, 9))
    nrm, rho, eta = rng.normal(size=(n_src, 3)), rng.normal(size=(n_src, 3)), 0.8
    trg_ids = np.concatenate([ids, -np.ones(n_extra, dtype=np.int32)])
    refs = {"sl": ps.pair_rows("sl", rs, f, rt), "dl9": ps.pair_rows("dl9", rs, f9, rt),
            "dl6": ps.pair_rows("dl6", rs, ps.double_layer_sym6(nrm, rho, eta), rt),
            "excl": ps.pair_rows("sl", rs, f, rt, src_ids=ids, trg_ids=trg_ids)}
    with skb.Context(1) as c:
        c.set_symmetric(0)
        c.set_targets(rt)
        c.set_sources(SL, rs)
        c.set_sources(DL, rs)
        c.set_source_normals(nrm)
        for T, S in TUNINGS:
            c.set_tuning(T, S)
            for mode in ("sl", "dl9", "dl6", "excl"):
                c.set_source_exclusion_ids(ids if mode == "excl" else None)
                call = {"sl": lambda: c.eval(SL, f), "dl9": lambda: c.eval(DL, f9),
                        "dl6": lambda: c.eval_double_layer(rho, eta), "excl": lambda: c.eval(SL, f)}[mode]
                u = _twice(call)
                K, _ = _plain_k(c, "sl" if mode in ("sl", "excl") else "dl9", n_trg, n_src, S)
                _check(f"plain {mode}", u, *refs[mode], K)


@pytest.mark.parametrize("kind", ["sl", "dl9"])
@pytest.mark.parametrize("n_src", [40001, 32767])
def test_plain_kernel_wide_reduce_one_target(kind, n_src):
    # n_trg = 1 against >= 32 767 sources: many splits and the wide reduce (256 splits of one tile at 32 767)
    rng = np.random.default_rng(3)
    rs, rt = rng.uniform(-2, 2, (n_src, 3)), rng.uniform(-2, 2, (1, 3))
    f = rng.normal(size=(n_src, 3 if kind == "sl" else 9))
    e, S = ps.pair_rows(kind, rs, f, rt)
    with skb.Context(1) as c:
        c.set_targets(rt)
        c.set_sources(SL if kind == "sl" else DL, rs)
        for Sreq in (0, 256, 7):
            c.set_tuning(0, Sreq)
            u = _twice(lambda: c.eval(SL if kind == "sl" else DL, f))
            K, p = _plain_k(c, kind, 1, n_src, Sreq)
            if Sreq == 256:
                assert p["n_splits"] == (256 if n_src == 32767 else 157) and p["n_splits"] >= 64
            _check(f"plain {kind} 1 x >= 32767", u, e, S, K)


@pytest.mark.parametrize("kind", ["sl", "dl9"])
def test_plain_kernel_planner_shape(kind):
    rng = np.random.default_rng(4)
    rs, rt = rng.uniform(-1, 1, (2500, 3)), rng.uniform(-1, 1, (3001, 3))
    f = rng.normal(size=(2500, 3 if kind == "sl" else 9))
    with skb.Context(1) as c:
        c.set_targets(rt)
        c.set_sources(SL if kind == "sl" else DL, rs)
        u = _twice(lambda: c.eval(SL if kind == "sl" else DL, f))
        K, p = _plain_k(c, kind, 3001, 2500)
    tile = 128 * p["T"]
    rows = ps.sample_rows(3001, (tile,), ragged_period=tile, full_limit=0)
    e, S = ps.pair_rows(kind, rs, f, rt, rows)
    _check(f"plain {kind} planner 3001 x 2500", u[rows], e, S, K)


def _single_pair_geometry(kind):
    rng = np.random.default_rng(5)
    lo, hi = (-150, 150) if kind == "sl" else (-55, 55)
    d = rng.normal(size=(600, 3))
    d *= (10.0 ** rng.uniform(lo, hi, 600) / np.linalg.norm(d, axis=1))[:, None]
    d = np.concatenate([d, [[2.0 ** -511, 0, 0], [0, 2.0 ** -511, 0], [2.0 ** -512, 0, 0], [0, 0, 2.0 ** -512],
                            [0, 0, 0]]]) if kind == "sl" else d
    far = np.array([[1e6, -1e6, 1e6]])
    e6 = rng.normal(size=(300, 3)) * (10.0 ** rng.uniform(-3, 3, 300))[:, None]
    return d, far, e6


@pytest.mark.parametrize("kind", ["sl", "dl9"])
def test_single_pair_rows(kind):
    """n_src <= 2: K is K_pair plus a few, where the rsqrt step is held tightly"""
    rng = np.random.default_rng(6)
    d, far, e6 = _single_pair_geometry(kind)
    fd = 3 if kind == "sl" else 9
    for rs, rt in ((np.zeros((1, 3)), d), (np.concatenate([far, far + 0.5]), far + e6)):
        f = rng.normal(size=(rs.shape[0], fd))
        e, S = ps.pair_rows(kind, rs, f, rt)
        with skb.Context(1) as c:
            c.set_targets(rt)
            c.set_sources(SL if kind == "sl" else DL, rs)
            for T in (1, 2, 4, 8):
                c.set_tuning(T, 0)
                u = _twice(lambda: c.eval(SL if kind == "sl" else DL, f))
                K, _ = _plain_k(c, kind, rt.shape[0], rs.shape[0])
                _check(f"plain {kind} single pair", u, e, S, K)
        if kind == "sl" and rs.shape[0] == 1:
            assert (u[-3:] == 0).all() and (u[-5:-3] != 0).all()   # |d|^2 = 2^-1024 and r = 0 give exactly 0


@pytest.mark.parametrize("kind", ["sl", "dl9"])
def test_cancellation_and_wide_range_rows(kind):
    rng = np.random.default_rng(7)
    fd = 3 if kind == "sl" else 9
    # +- pairs about each of 6 targets, opposite Stokeslet strengths / equal stresslet strengths: exact row ~ 0
    ctr = rng.uniform(-1, 1, (6, 3))
    src, fs = [], []
    for c0 in ctr:
        dl = rng.normal(size=(100, 3)) * (10.0 ** rng.uniform(-2, 0, 100))[:, None]
        fv = rng.normal(size=(100, fd))
        src += [c0 + dl, c0 - dl]
        fs += [fv, -fv if kind == "sl" else fv]
    # a few near sources, thousands far: the far rows' S is far below the near rows'
    src.append(rng.normal(size=(5, 3)) * 0.01)
    fs.append(rng.normal(size=(5, fd)) * 1e3)
    src.append(rng.normal(size=(3000, 3)) + 1e3)
    fs.append(rng.normal(size=(3000, fd)))
    rs, f = np.concatenate(src), np.concatenate(fs)
    rt = np.concatenate([ctr, rng.normal(size=(200, 3)) * 0.05, rng.normal(size=(300, 3)) - 1e4])
    e, S = ps.pair_rows(kind, rs, f, rt)
    with skb.Context(1) as c:
        c.set_targets(rt)
        c.set_sources(SL if kind == "sl" else DL, rs)
        for T in (0, 1, 8):
            c.set_tuning(T, 0)
            u = _twice(lambda: c.eval(SL if kind == "sl" else DL, f))
            K, _ = _plain_k(c, kind, rt.shape[0], rs.shape[0])
            _check(f"plain {kind} cancellation / wide range", u, e, S, K)


# ---- symmetric kernel ---------------------------------------------------------------------------------------------
def _sym_eval(rs, rt, f, ids=None, part=None):
    with skb.Context(1) as c:
        c.set_symmetric(1)
        if part is not None:
            c.set_sym_partition(*part)
        c.set_targets(rt)
        c.set_sources(SL, rs)
        if ids is not None:
            c.set_source_exclusion_ids(ids)
        u = _twice(lambda: c.eval(SL, f))
        assert c.last_eval_was_symmetric()
    return u


# (the symmetric path needs at least two 1024-node blocks of sources: below that the plain kernel serves the call)
@pytest.mark.parametrize("n_src,n_extra", [(2048, 0), (2049, 300), (3071, 0), (4097, 4097)])
def test_symmetric_kernel(n_src, n_extra):
    rng = np.random.default_rng(10 + n_src)
    rs = rng.uniform(-1, 1, (n_src, 3))
    rt = np.concatenate([rs, rng.uniform(-1, 1, (n_extra, 3))])
    f = rng.normal(size=(n_src, 3))
    rows = ps.sample_rows(rt.shape[0], (ps.SYM_BLOCK, ps.SYM_GROUP), n_lead=n_src, ragged_period=ps.SYM_GROUP,
                          full_limit=1024)
    e_b, S_b = ps.pair_blocks("sl", rs, f, rt, rows, block=ps.SYM_BLOCK)
    nb = ps.n_pad(n_src) // ps.SYM_BLOCK
    lead = rows[rows < n_src]
    for parts in ([(0, 1)] + ([(p, n) for n in (2, 3) for p in range(n)] if n_src == 4097 else [])):
        m = ps.sym_part_mult(rows, n_src, *parts)
        K = ps.k_sym_rows(n_src, rt.shape[0], rows, *parts, plan=capi.sym_plan_query(nb, *parts, num_sms=_num_sms()))
        e, S = ps.combine(e_b, m), ps.combine(S_b, np.abs(m))
        u = _sym_eval(rs, rt, f, part=parts if parts[1] > 1 else None)
        _check(f"symmetric{' partition' if parts[1] > 1 else ''}", u[rows], e, S, K)
        if n_extra and parts == (0, 1):   # the same leading rows without remainder targets
            u0 = _sym_eval(rs, rs, f)
            k_lead = K[rows < n_src]
            _check("symmetric", u0[lead], e[rows < n_src], S[rows < n_src], k_lead)


def test_symmetric_kernel_duplicates_zero_strengths_and_exclusion():
    rng = np.random.default_rng(20)
    base = rng.uniform(-1, 1, (1100, 3))
    rs = np.repeat(base, 2, axis=0)[:2199]          # every node twice: r == 0 pairs off the diagonal
    n_src = rs.shape[0]
    rt = np.concatenate([rs, rng.uniform(-1, 1, (150, 3))])
    f = rng.normal(size=(n_src, 3))
    f[::7] = 0.0
    ids = np.repeat(np.arange(n_src), rng.choice([5, 16, 37], size=n_src))[:n_src].astype(np.int32)
    trg_ids = np.concatenate([ids, -np.ones(150, dtype=np.int32)])
    rows = ps.sample_rows(rt.shape[0], (ps.SYM_BLOCK, ps.SYM_GROUP), n_lead=n_src, ragged_period=ps.SYM_GROUP,
                          full_limit=1024)
    plan = capi.sym_plan_query(ps.n_pad(n_src) // ps.SYM_BLOCK, num_sms=_num_sms())
    K = ps.k_sym_rows(n_src, rt.shape[0], rows, plan=plan)
    _check("symmetric duplicates", _sym_eval(rs, rt, f)[rows], *ps.pair_rows("sl", rs, f, rt, rows), K)
    _check("symmetric exclusion", _sym_eval(rs, rt, f, ids=ids)[rows],
           *ps.pair_rows("sl", rs, f, rt, rows, src_ids=ids, trg_ids=trg_ids), K)


# ---- cross kernel -------------------------------------------------------------------------------------------------
def test_cross_kernel_each_direction(monkeypatch):
    from test_gpu_flow import ft_of, load, make_system
    monkeypatch.setenv("SKB_SYMMETRIC", "1")
    fib, shell, body = make_system(30, 70, 700, 0, 0, nodes=(16, 24, 40, 56))
    n_fib, n_sh = fib["pos"].shape[0], shell["pos"].shape[0]
    assert n_fib >= 2048 and n_fib % ps.CROSS_BLOCK, n_fib       # the cross kernel runs, with a tail
    eta = 0.7
    h = ps.weighted_forces(fib["forces"], ps.trapezoid_weights(fib["n_nodes"], fib["lengths"]))
    s6 = ps.double_layer_sym6(shell["normals"], shell["density"], eta)
    e_sh, S_sh = ps.pair_rows("sl", fib["pos"], h, shell["pos"], scale=ps.scale_of("sl", eta))
    rows = ps.sample_rows(n_fib, (ps.CROSS_BLOCK, ps.SYM_GROUP), ragged_period=ps.SYM_GROUP, full_limit=0)
    e_f, S_f = ps.pair_rows("dl6", shell["pos"], s6, fib["pos"], rows, scale=ps.scale_of("dl6", eta))
    zf, zs = np.zeros_like(fib["forces"]), np.zeros_like(shell["density"])
    launches = {}
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        for cross in (1, 0):
            fl.set_cross(cross)
            v_sh = _twice(lambda: fl.matvec(fib["forces"], zs, body["density"], ft_of(body), eta))
            launches[cross] = fl.stats()["launches"]
            v_f = _twice(lambda: fl.matvec(zf, shell["density"], body["density"], ft_of(body), eta))
            k_sh = ps.k_cross("sl", n_fib) if cross else ps.k_plain_bound("sl", n_fib)
            k_f = ps.k_cross("dl6", n_sh) if cross else ps.k_plain_bound("dl6", n_sh)
            tag = "cross" if cross else "plain (cross off)"
            _check(f"{tag} periphery rows", v_sh[n_fib:], e_sh, S_sh, k_sh)
            _check(f"{tag} fiber rows", v_f[rows], e_f, S_f, k_f)
    assert launches[1] != launches[0]


def test_worst_ratios_report():
    print("\nworst ratio / K:")
    for k, v in sorted(WORST.items()):
        print(f"    {k:42s} {v:.3g}")

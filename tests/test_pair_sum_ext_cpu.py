"""CPU tests of the row-wise criterion of tests/pair_sum_reference.py, which tests/test_gpu_pair_sum_ext.py applies to
the plain, symmetric and cross pair kernels on the device: |dev - ext| <= K u S per row component, ext the restatement
in np.longdouble, S the same sum on absolute values, K fixed from the kernel source (the module's docstring derives it).

The criterion is attainable: a float64 emulation of the kernels' pair arithmetic, in stokeslet_chains' and
stresslet_chains' instruction order with the rsqrt seed perturbed to the edge of its error, meets K_pair on every pair
(random pairs, |d| near 2^-511 where r^2 meets DBL_MIN, separations over 1e-150 .. 1e150), and float64 sums of those
terms in several orders meet K.  It is sharp: every planted defect misses its bound on the shape that targets it (the
printed margins; all but the second-order Newton step miss by more than DEFECT_FACTOR).  The restatement is the
operation of the project's long-double oracle, and the row sampler returns every structural edge of a plan."""
import numpy as np
import pytest

import oracle as orc
import pair_sum_reference as ps
from skellysim_b200 import capi

DEFECT_FACTOR = 1e6
RNG = np.random.default_rng


def _pairs(rng, n, log_sep=(-0.5, 0.5), centre=1.0):
    t = rng.uniform(-centre, centre, (n, 3))
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    return t, t - u * (10.0 ** rng.uniform(*log_sep, n))[:, None]


def _strengths(rng, kind, n):
    return rng.normal(size=(n, {"sl": 3, "dl6": 6, "dl9": 9}[kind]))


def _pair_ratio(kind, t, s, f, eta, defect=None):
    """per-pair |term - ext| / (u S)"""
    got = ps.pair_terms_f64(kind, t, s, f, eta, defect)
    return ps.ratio(got, *ps.pair_terms_ext(kind, t, s, f)).max(axis=1)


@pytest.mark.parametrize("kind", ["sl", "dl9"])
def test_pair_arithmetic_meets_k_pair(kind):
    assert np.finfo(np.longdouble).nmant >= 63
    rng = RNG(1 if kind == "sl" else 2)
    worst = 0.0
    n = 5000
    for log_sep, centre in (((-0.5, 0.5), 1.0), ((-3, 3), 1.0), ((-1, 1), 1e6), ((-6, -5), 1e6)):
        t, s = _pairs(rng, n, log_sep, centre)
        f = _strengths(rng, kind, n)
        for eta in (ps.SEED_REL, -ps.SEED_REL, rng.uniform(-ps.SEED_REL, ps.SEED_REL, n)):
            r = _pair_ratio(kind, t, s, f, eta)
            assert np.isfinite(r).all() and (r <= ps.K_PAIR[kind]).all(), (log_sep, centre, r.max())
            worst = max(worst, r.max())
    print(f"\n{kind}: float64 pair terms, worst ratio {worst:.2f} (K_pair {ps.K_PAIR[kind]})")


@pytest.mark.parametrize("kind", ["sl", "dl9"])
def test_pair_arithmetic_at_the_extremes(kind):
    rng = RNG(3)
    # separations over 1e-150 .. 1e150 (the stresslet's y^5 stays normal only within about 1e-61 .. 1e61)
    lo, hi = (-150, 150) if kind == "sl" else (-55, 55)
    t, s = _pairs(rng, 4000, (lo, hi))
    # |d| near 2^-511: r^2 at DBL_MIN, both sides (the Stokeslet only: the stresslet's y^5 overflows there)
    if kind == "sl":
        k = np.arange(400)
        t2 = rng.uniform(-1e-300, 1e-300, (400, 3))
        dx = 2.0 ** -511 * (1 + (k - 200) * 2.0 ** -40)
        t, s = np.concatenate([t, t2]), np.concatenate([s, t2 - np.stack([dx, 0 * dx, 0 * dx], 1)])
    f = _strengths(rng, kind, t.shape[0])
    for eta in (ps.SEED_REL, -ps.SEED_REL):
        r = _pair_ratio(kind, t, s, f, eta)
        assert np.isfinite(r).all() and (r <= ps.K_PAIR[kind]).all(), r.max()


def test_the_r0_rule_is_decided_on_the_float64_r2():
    # |d|^2 = 2^-1022 exactly is evaluated, |d|^2 = 2^-1024 gives exactly 0, and so does r = 0
    t = np.array([[0.0, 0.0, 0.0]])
    for dx, live in ((2.0 ** -511, True), (2.0 ** -512, False), (0.0, False)):
        e, S = ps.pair_rows("sl", np.array([[dx, 0.0, 0.0]]), np.ones((1, 3)), t)
        assert (e != 0).any() == live and (S != 0).any() == live
        got = ps.pair_terms_f64("sl", t, np.array([[dx, 0.0, 0.0]]), np.ones((1, 3)), 0.0)
        assert (got != 0).any() == live
    # a pair whose float64 r^2 rounds up to DBL_MIN although its exact r^2 is below: evaluated, as on the device
    d = np.nextafter(2.0 ** -511, 0.0)
    assert d * d < ps.DBL_MIN and ps.r2_kernel(np.float64(d), np.float64(0), np.float64(0)) < ps.DBL_MIN
    a = 2.0 ** -511 * np.sqrt(0.5)
    r2 = ps.r2_kernel(np.float64(a), np.float64(a), np.float64(0.0))
    e, _ = ps.pair_rows("sl", np.array([[a, a, 0.0]]), np.ones((1, 3)), t)
    assert (e != 0).any() == (r2 >= ps.DBL_MIN)


@pytest.mark.parametrize("kind", ["sl", "dl9"])
def test_float64_sums_in_any_order_meet_k(kind):
    rng = RNG(4)
    n = 1500
    s = rng.uniform(-1, 1, (n, 3))
    t = np.repeat(rng.uniform(-1, 1, (1, 3)), n, axis=0)
    f = _strengths(rng, kind, n)
    terms = ps.pair_terms_f64(kind, t, s, f, rng.uniform(-ps.SEED_REL, ps.SEED_REL, n))
    e, S = ps.pair_rows(kind, s, f, t[:1])
    scale = (1.0 if kind == "sl" else -3.0) / (8.0 * np.pi)
    n_splits = 12
    per = -(-n // n_splits)
    orders = {"sequential": np.arange(n), "reversed": np.arange(n)[::-1]}
    sums = {k: ps.accumulate(terms, o) for k, o in orders.items()}
    parts = [ps.accumulate(terms, np.arange(a, min(n, a + per))) for a in range(0, n, per)]
    sums["splits"] = ps.accumulate(np.array(parts, dtype=ps.LD), range(len(parts)))
    for k in range(3):                                       # random binary trees
        v = [x.astype(np.float64) for x in terms]
        while len(v) > 1:
            i, j = sorted(rng.choice(len(v), 2, replace=False))
            a = v.pop(j)
            v[i] = v[i] + a
        sums[f"tree{k}"] = v[0]
    K = ps.k_plain(kind, n, -(-n // 128), n_splits)
    for name, u in sums.items():
        r = ps.ratio(u * scale, e[0], S[0]).max()
        assert r <= K, (name, r, K)


# ---- the planted defects -------------------------------------------------------------------------------------------
def _plain_case(rng, kind, n_src, n_extra, ids=False):
    rs = rng.uniform(-1, 1, (n_src, 3))
    rt = np.concatenate([rs, rng.uniform(-1, 1, (n_extra, 3))])
    f = _strengths(rng, kind, n_src)
    kw = {}
    if ids:
        n_nodes = rng.choice([5, 8, 13, 21], size=n_src)
        src_ids = np.repeat(np.arange(n_src), n_nodes)[:n_src]
        kw = dict(src_ids=src_ids, trg_ids=np.concatenate([src_ids, -np.ones(n_extra, dtype=int)]))
    return rs, f, rt, kw


def _miss(kind, rs, f, rt, K, defect, rows=None, **kw):
    e, S = ps.pair_rows(kind, rs, f, rt, rows, **kw)
    bad, _ = ps.pair_rows(kind, rs, f, rt, rows, defect=defect, **kw)
    return float(np.max(ps.ratio(bad.astype(np.float64), e, S) / K))


def test_newton2_is_caught_on_single_pair_rows():
    rng = RNG(5)
    t, s = _pairs(rng, 2000)
    f = _strengths(rng, "sl", 2000)
    K = ps.k_plain("sl", 1, 1, 1)
    worst = 0.0
    for eta in (ps.SEED_REL, -ps.SEED_REL):
        e, S = ps.pair_terms_ext("sl", t, s, f)
        bad = ps.pair_terms_f64("sl", t, s, f, eta, "newton2")
        worst = max(worst, float(np.max(ps.ratio(bad, e, S)) / K))
    print(f"\nnewton2 on single-pair rows: misses its bound by {worst:.3g} x K (K = {K})")
    assert worst > 1.5


def test_subnormal_rule_defect():
    t = np.zeros((1, 3))
    f = np.ones((2, 3))
    rs = np.array([[2.0 ** -512, 0.0, 0.0], [1.0, 0.5, 0.25]])
    m = _miss("sl", rs, f, t, ps.k_plain("sl", 2, 1, 1), "no_subnormal_rule")
    print(f"\nno_subnormal_rule: misses by {m:.3g} x K")
    assert m > DEFECT_FACTOR


@pytest.mark.parametrize("defect,n_src", [("odd_source_dropped", 129), ("odd_source_dropped", 333),
                                          ("ragged_tile_dropped", 129), ("split_dropped", 40001)])
def test_plain_structure_defects(defect, n_src):
    rng = RNG(6)
    n_trg = 1 if defect == "split_dropped" else 300
    rs, f, rt, _ = _plain_case(rng, "sl", n_src, n_trg)
    rows = np.arange(n_src, n_src + n_trg)
    p = capi.plan_query(0, n_trg, n_src)
    K = ps.k_plain("sl", n_src, p["tiles_per_split"], p["n_splits"])
    sel = ps.source_select(n_src, defect, p["tiles_per_split"], p["n_splits"])
    e, S = ps.pair_rows("sl", rs, f, rt, rows)
    bad, _ = ps.pair_rows("sl", rs, f, rt, rows, select=sel)
    m = float(np.max(ps.ratio(bad.astype(np.float64), e, S) / K))
    print(f"\n{defect} at n_src {n_src} ({p['n_splits']} splits): misses by {m:.3g} x K")
    assert m > DEFECT_FACTOR


@pytest.mark.parametrize("defect", ["sym6_doubled", "stresslet_sign"])
def test_stresslet_defects(defect):
    rng = RNG(7)
    rs, f, rt, _ = _plain_case(rng, "dl9", 129, 200)
    m = _miss("dl9", rs, f, rt, ps.k_plain_bound("dl9", 129), defect)
    print(f"\n{defect}: misses by {m:.3g} x K")
    assert m > DEFECT_FACTOR


def test_exclusion_by_position_defect():
    rng = RNG(8)
    rs, f, rt, kw = _plain_case(rng, "sl", 500, 77, ids=True)
    m = _miss("sl", rs, f, rt, ps.k_plain_bound("sl", 500), "excl_by_position", **kw)
    print(f"\nexcl_by_position: misses by {m:.3g} x K")
    assert m > DEFECT_FACTOR


@pytest.mark.parametrize("defect,n_parts", [("diag_reverse_counted", 1), ("item_reverse_dropped", 1),
                                            ("serpentine_flipped", 3), ("diag_reverse_counted", 2)])
def test_symmetric_structure_defects(defect, n_parts):
    rng = RNG(9)
    n_src = 4097
    rs = rng.uniform(-1, 1, (n_src, 3))
    f = _strengths(rng, "sl", n_src)
    nb = ps.n_pad(n_src) // ps.SYM_BLOCK
    rows = ps.sample_rows(n_src, (ps.SYM_BLOCK, ps.SYM_GROUP), ragged_period=ps.SYM_GROUP, n_random=64)
    e_b, S_b = ps.pair_blocks("sl", rs, f, rs, rows, block=ps.SYM_BLOCK)
    m = 0.0
    for part in range(n_parts):
        plan = capi.sym_plan_query(nb, part, n_parts)
        item = None
        if defect == "item_reverse_dropped":
            gpb = capi.sym_groups_per_block()
            item = next(it[:3] for it in plan[0] if it[1] >= gpb * (it[0] + 1))
            rows_i = np.arange(item[1] * ps.SYM_GROUP, min(n_src, item[2] * ps.SYM_GROUP))
            e_b, S_b = ps.pair_blocks("sl", rs, f, rs, rows_i, block=ps.SYM_BLOCK)
            rows = rows_i
        good = ps.sym_part_mult(rows, n_src, part, n_parts)
        bad = ps.sym_part_mult(rows, n_src, part, n_parts, defect, item)
        K = ps.k_sym_rows(n_src, n_src, rows, part, n_parts, plan)
        e, S = ps.combine(e_b, good), ps.combine(S_b, np.abs(good))
        r = ps.ratio(ps.combine(e_b, bad).astype(np.float64), e, S) / K[:, None]
        m = max(m, float(np.max(r)))
    print(f"\n{defect} over {n_parts} part(s): misses by {m:.3g} x K")
    assert m > DEFECT_FACTOR


def test_cross_tail_defect():
    rng = RNG(10)
    n_fib, n_sh = 1100, 300
    rf = rng.uniform(-1, 1, (n_fib, 3))
    rsh = rng.normal(size=(n_sh, 3)) * 3
    h = _strengths(rng, "sl", n_fib)
    K = ps.k_cross("sl", n_fib)
    e, S = ps.pair_rows("sl", rf, h, rsh)
    bad, _ = ps.pair_rows("sl", rf, h, rsh, select=ps.cross_tail_select(n_fib))
    m = float(np.max(ps.ratio(bad.astype(np.float64), e, S) / K))
    print(f"\ncross_tail_acts: misses by {m:.3g} x K")
    assert m > DEFECT_FACTOR


# ---- structure restatements against the host planners ---------------------------------------------------------------
@pytest.mark.parametrize("nb,n_parts", [(5, 1), (5, 2), (5, 3), (9, 3)])
def test_sym_owner_and_partials_follow_the_planner(nb, n_parts):
    seen = []
    for part in range(n_parts):
        items, row_begin = capi.sym_plan_query(nb, part, n_parts)
        owned = sorted({it[0] for it in items})
        assert owned == [I for I in range(nb) if ps.sym_row_owner(I, n_parts) == part]
        seen += owned
        parts = ps.sym_partials(nb * ps.SYM_BLOCK, part, n_parts, (items, row_begin))
        for b in range(nb):
            n_items = row_begin[b + 1] - row_begin[b]
            assert parts[b] == n_items + sum(1 for I in owned if I < b)
    assert sorted(seen) == list(range(nb))
    # the parts' multipliers tile the full sum exactly once
    rows = np.arange(0, nb * ps.SYM_BLOCK, 97)
    tot = sum(ps.sym_part_mult(rows, nb * ps.SYM_BLOCK, p, n_parts) for p in range(n_parts))
    assert (tot == 1).all()


@pytest.mark.parametrize("n_trg,n_src", [(1037, 129), (3000, 2500), (1, 40000), (8000, 300), (5000, 4097)])
def test_row_sampler_returns_every_structural_edge(n_trg, n_src):
    for T in (1, 2, 4, 8):
        p = capi.plan_query(0, n_trg, n_src, force_T=T)
        tile = 128 * p["T"]
        rows = set(ps.sample_rows(n_trg, (tile,), ragged_period=tile).tolist())
        assert len(rows) == n_trg or len(rows) < n_trg
        for x in range(p["grid_x"]):
            a, b = x * tile, min(n_trg, (x + 1) * tile) - 1
            assert a in rows and b in rows
        last = (p["grid_x"] - 1) * tile
        if n_trg - last < tile:
            assert set(range(last, n_trg)) <= rows
    # symmetric: block and group edges of the leading rows, the ragged last group, the remainder rows' tiles
    rows = set(ps.sample_rows(n_trg + n_src, (ps.SYM_BLOCK, ps.SYM_GROUP), n_lead=n_src,
                              ragged_period=ps.SYM_GROUP).tolist())
    for per in (ps.SYM_BLOCK, ps.SYM_GROUP):
        for a in range(0, n_src, per):
            assert a in rows and min(n_src, a + per) - 1 in rows
    if n_src % 32:
        assert set(range(n_src // 32 * 32, n_src)) <= rows
    for T in (1, 2, 4, 8):
        for a in range(n_src, n_src + n_trg, 128 * T):
            assert a in rows and min(n_src + n_trg, a + 128 * T) - 1 in rows
    assert len(rows) >= min(n_trg + n_src, 256)


def test_ext_agrees_with_the_long_double_oracle():
    rng = RNG(11)
    rs, rt = rng.uniform(-1, 1, (700, 3)), rng.uniform(-1, 1, (300, 3))
    for kind, fn in (("sl", orc.stokeslet_direct_ld), ("dl9", orc.stresslet_direct_ld)):
        f = _strengths(rng, kind, 700)
        e, S = ps.pair_rows(kind, rs, f, rt)
        r = ps.ratio(fn(rs, f, rt), e, S).max()
        print(f"\n{kind}: oracle vs ext {r:.3g} u S")
        assert r <= 2.0


def test_packed_strengths_are_the_devices_float64():
    # the double layer's sym6 is pack_dl9 of the host-formed 2 eta n (x) rho (pack_dl_normal_density_kernel's claim)
    rng = RNG(12)
    n, rho, eta = rng.normal(size=(50, 3)), rng.normal(size=(50, 3)), 0.7
    f9 = orc.form_double_layer(n, rho, eta)
    s6 = ps.double_layer_sym6(n, rho, eta)
    ref = np.stack([f9[:, 0], f9[:, 4], f9[:, 8], f9[:, 1] + f9[:, 3], f9[:, 2] + f9[:, 6], f9[:, 5] + f9[:, 7]], 1)
    assert np.array_equal(s6, ref)
    w = ps.trapezoid_weights([5, 9], [1.3, 0.7])
    ref = np.concatenate([orc.trapezoid_weights(5, 1.3), orc.trapezoid_weights(9, 0.7)])
    assert np.allclose(w, ref, rtol=1e-15, atol=0)

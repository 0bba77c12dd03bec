"""The criterion of tests/gradient_reference.py is attainable and sharp, without a GPU.

Attainable: a float64 emulation of stokeslet_grad_source and stresslet_grad_source, in their instruction order with the
rsqrt seed perturbed to +-2^-22.4, meets K_pair on every pair at separations from 1e-40 to 1e40, each pair's target
placed at up to 1e3 times its separation so that no pair is lost to rounding (none is masked; worst measured ratio 9.4
of 56 for the Stokeslet, 11.4 of 77 for the stresslet), and its pairs are exactly 0 where the float64 r^2 is just
below DBL_MIN.  Float64 sums of those chains in several orders (sequential, reversed, in splits reduced and scaled)
meet k_pair, and float64 restatements of oseen_grad_add_kernel and rotlet_grad_add_kernel (contracted r^2, every other
operation rounded on its own) meet k_points and k_rotlet on rows that reach their eps edges.  Worst ratios / K,
printed by the tests: the sums 0.0013 (Stokeslet) and 0.0012 (stresslet), the Oseen gradient 0.10, the rotlet
gradient 0.19.

The regularised branches (r <= EPS for the Oseen gradient, r^2 < EPS2 for the rotlet) are the derivative of the
oracle's regularised velocities: long-double central differences with h = 1e-9 at r from 1e-7 to 9e-6, where both
points stay inside the branch.

Sharp: each planted defect of gradient_reference.DEFECTS misses its bound on some row of one edge case by more than
MISS K; where only the row exactly at an eps edge can see a defect, the case is shown to hold that row.
"""
import numpy as np
import pytest

import flow_reference as fr
import gradient_reference as gr
import oracle as orc
import pair_sum_reference as ps
from test_flow_ext_cpu import BG, edge_fibers, point_sources, shell_and_bodies

MISS = 1e9
RNG = np.random.default_rng


# ---- edge geometry, shared with tests/test_gpu_listener_gradient_ext.py ---------------------------------------------
def last_regularised(rule):
    """the largest float64 offset dx along an axis for which rule(float64 r^2 of (dx, 0, 0)) still regularises"""
    dx = np.float64(fr.EPS)
    while rule(dx * dx):
        dx = np.nextafter(dx, 1.0)
    while not rule(dx * dx):
        dx = np.nextafter(dx, 0.0)
    return dx


OSEEN_RULE = lambda r2: np.sqrt(r2) <= fr.EPS   # noqa: E731  (oseen_grad_add_kernel)
ROTLET_RULE = lambda r2: r2 < fr.EPS2           # noqa: E731  (rotlet_grad_add_kernel)
OSEEN_LAST = last_regularised(OSEEN_RULE)
ROTLET_LAST = last_regularised(ROTLET_RULE)
SUBNORMAL = (1e-160, -3e-158)                   # offsets whose r^2 is subnormal


def _axis(p, dxs):
    return np.asarray(p, dtype=np.float64) + np.array([[dx, 0.0, 0.0] for dx in dxs])


def inside_eps(rng, centres, n):
    """n targets at r from 1e-7 to 9e-6 from each of the centres, random directions"""
    out = []
    for p in centres:
        u = rng.normal(size=(n, 3))
        u /= np.linalg.norm(u, axis=1)[:, None]
        out.append(p + u * rng.uniform(1e-7, 9e-6, (n, 1)))
    return np.concatenate(out)


def edge_targets(rng, fib, shell, body, pts, n_free=150):
    """free targets; targets on every fiber, shell and body node, point source and body centre; at subnormal-r^2
    offsets from fiber node 0 (x == 0); at the last regularised offset of each rule and the next float64 beyond it,
    both signs, along x from the point sources and the body centre whose x is 0 (dy = dz = 0: every form of r^2 exact);
    at EPS exactly; and strictly inside eps"""
    edges = [OSEEN_LAST, np.nextafter(OSEEN_LAST, 1.0), ROTLET_LAST, np.nextafter(ROTLET_LAST, 1.0), fr.EPS]
    out = [rng.uniform(-2.5, 2.5, (n_free, 3)), fib["pos"], shell["pos"], body["pos"], pts, body["centers"]]
    assert fib["pos"][0][0] == 0.0
    out.append(_axis(fib["pos"][0], SUBNORMAL))
    for p in list(pts[:2]) + [body["centers"][0]]:
        assert p[0] == 0.0
        out.append(_axis(p, [s * e for e in edges for s in (1, -1)]))
    out.append(inside_eps(rng, list(pts) + [body["centers"][0]], 4))
    return np.concatenate(out)


def edge_case(seed, nodes=(8, 16, 31), n_shell=120, per=40, n_free=150):
    rng = RNG(seed)
    fib = edge_fibers(rng, nodes)
    shell, body = shell_and_bodies(rng, n_shell, per)
    points = point_sources(rng)
    return fib, shell, body, points, edge_targets(rng, fib, shell, body, points[0], n_free)


def branch_rows(r, fib, shell, body, pts):
    """the rows of each branch the edge targets are there to reach, decided as the kernels decide them"""
    r = np.asarray(r, dtype=np.float64)

    def r2(src):
        d = r[:, None, :] - np.asarray(src, dtype=np.float64)[None, :, :]
        return ps.r2_kernel(d[..., 0], d[..., 1], d[..., 2])
    out = {f"r == 0 on {k}": (r2(s) == 0).any(axis=1)
           for k, s in (("fiber nodes", fib["pos"]), ("shell nodes", shell["pos"]), ("body nodes", body["pos"]),
                        ("point sources", pts), ("body centres", body["centers"]))}
    out["subnormal r^2 to a fiber node"] = ((r2(fib["pos"]) > 0) & (r2(fib["pos"]) < ps.DBL_MIN)).any(axis=1)
    for name, src, rule, last in (("Oseen, points", pts, OSEEN_RULE, OSEEN_LAST),
                                  ("rotlet, points", pts, ROTLET_RULE, ROTLET_LAST),
                                  ("rotlet, body centres", body["centers"], ROTLET_RULE, ROTLET_LAST)):
        q = r2(src)
        out[f"{name}: regularised at the edge"] = (rule(q) & (q == last * last)).any(axis=1)
        out[f"{name}: not regularised one ulp beyond"] = \
            (~rule(q) & (q == np.nextafter(last, 1.0) ** 2)).any(axis=1)
        out[f"{name}: strictly inside eps"] = (rule(q) & (q > 0) & (q < 1e-10)).any(axis=1)
    q = r2(pts)
    out["Oseen, points: float64 r == EPS"] = (np.sqrt(q) == fr.EPS).any(axis=1)
    out["rotlet, points: float64 r^2 == EPS2"] = (q == fr.EPS2).any(axis=1)
    return out


# ---- attainable ---------------------------------------------------------------------------------------------------
def _pairs(rng, n, log_sep, centre=1.0):
    """n pairs at separations 10^log_sep; t uniform in [-centre, centre], or (centre None) at up to 1e3 times each
    pair's own separation, so that no separation is lost to the rounding of t - u sep"""
    sep = 10.0 ** rng.uniform(*log_sep, n)
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    scale = centre if centre is not None else (sep * 10.0 ** rng.uniform(0, 3, n))[:, None]
    t = rng.uniform(-1, 1, (n, 3)) * scale
    return t, t - u * sep[:, None]


@pytest.mark.parametrize("kind", ["sl", "dl6"])
def test_pair_chains_meet_k_pair(kind):
    assert np.finfo(np.longdouble).nmant >= 63
    rng = RNG(1 if kind == "sl" else 2)
    dim = 3 if kind == "sl" else 6
    worst = 0.0
    n = 4000
    for log_sep, centre in (((-0.5, 0.5), 1.0), ((-3, 3), 1e3), ((-40, 40), None), ((-40, -38), None),
                            ((-20, -10), None), ((38, 40), None), ((38, 40), 1.0)):
        t, s = _pairs(rng, n, log_sep, centre)
        d = t - s
        assert (ps.r2_kernel(d[:, 0], d[:, 1], d[:, 2]) >= ps.DBL_MIN).all()   # no pair masked: every chain runs
        f = rng.normal(size=(n, dim))
        ext, S = gr.pair_grad_ext(kind, t, s, f)
        for eta in (ps.SEED_REL, -ps.SEED_REL, rng.uniform(-ps.SEED_REL, ps.SEED_REL, n)):
            g = gr.add_pair_f64(kind, np.zeros((n, 10)), t, s, f, eta)
            r = gr.ratio(g, ext, S)
            assert np.isfinite(g).all() and (r <= gr.K_PAIR_GRAD[kind]).all(), (log_sep, centre, r.max())
            worst = max(worst, float(r.max()))
    # r^2 just below DBL_MIN: the pair is masked and adds exactly 0, on the device and in ext (at r^2 = DBL_MIN itself
    # y^3 overflows: outside the domain)
    k = np.arange(1, 200)
    t = rng.uniform(-1e-300, 1e-300, (k.size, 3))
    dx = np.sqrt(ps.DBL_MIN) * (1 - k * 2.0 ** -45)
    s = t - np.stack([dx, 0 * dx, 0 * dx], 1)
    assert (ps.r2_kernel(t[:, 0] - s[:, 0], t[:, 1] - s[:, 1], t[:, 2] - s[:, 2]) < ps.DBL_MIN).all()
    f = rng.normal(size=(k.size, dim))
    ext, S = gr.pair_grad_ext(kind, t, s, f)
    for eta in (ps.SEED_REL, -ps.SEED_REL):
        assert (gr.add_pair_f64(kind, np.zeros((k.size, 10)), t, s, f, eta) == 0).all() and (ext == 0).all()
    print(f"\n{kind}: float64 gradient chains, worst ratio {worst:.3g} (K_pair {gr.K_PAIR_GRAD[kind]})")


@pytest.mark.parametrize("kind", ["sl", "dl6"])
def test_float64_sums_in_several_orders_meet_k(kind):
    rng = RNG(4)
    n, n_splits, eta = 1500, 12, 0.37
    dim = 3 if kind == "sl" else 6
    s = rng.uniform(-1, 1, (n, 3))
    t = rng.uniform(-1, 1, (3, 3))
    f = rng.normal(size=(n, dim)) * 10.0 ** rng.uniform(-3, 3, (n, 1))
    seed_err = rng.uniform(-ps.SEED_REL, ps.SEED_REL, n)
    ext, S, K = gr.pair_grad_rows(kind, s, f, t, eta)
    scale = 1.0 / eta * ((1.0 if kind == "sl" else -3.0) / (8.0 * np.pi))

    def walk(order):
        g = np.zeros((len(t), 10))
        for j in order:
            g = gr.add_pair_f64(kind, g, t, np.repeat(s[j:j + 1], len(t), 0), np.repeat(f[j:j + 1], len(t), 0),
                                seed_err[j])
        return g
    per = -(-n // n_splits)
    sums = {"sequential": walk(range(n)) * scale, "reversed": walk(range(n - 1, -1, -1)) * scale}
    acc = np.zeros((len(t), 10))
    for a in range(0, n, per):
        acc = acc + walk(range(a, min(n, a + per)))
    sums["splits"] = acc * scale
    worst = 0.0
    for name, g in sums.items():
        r = gr.ratio(g, ext, S) / K[:, None]
        assert (r <= 1).all(), (name, r.max())
        worst = max(worst, float(r.max()))
    print(f"\n{kind}: float64 sums, worst ratio / K {worst:.3g} (K {K[0]:.0f})")


def _oseen_grad_f64(t, pts, f, eta):
    """oseen_grad_add_kernel in float64: contracted r^2 and dr dr + reg2 (as built), the rest rounded on its own"""
    c = 1.0 / (8.0 * np.pi * eta)
    acc = np.zeros((len(t), 10))
    for s in range(len(pts)):
        d = t - pts[s]
        dr = np.sqrt(ps.r2_kernel(d[:, 0], d[:, 1], d[:, 2]))
        with np.errstate(divide="ignore", invalid="ignore"):
            D = np.where(dr > fr.EPS, dr, np.sqrt(ps.fma(dr, dr, fr.REG2)))
            g3 = 1.0 / ((D * D) * D)
            hr = (3.0 * g3) / (D * D)
        fs = f[s]
        rf = (d[:, 0] * fs[0] + d[:, 1] * fs[1]) + d[:, 2] * fs[2]
        a = np.zeros((len(t), 10))
        for i in range(3):
            for j in range(3):
                inner = ((rf if i == j else 0.0) + d[:, i] * fs[j]) - fs[i] * d[:, j]
                a[:, 3 * i + j] = g3 * inner - ((hr * rf) * d[:, i]) * d[:, j]
        a[:, 9] = (2.0 * g3) * rf
        a[dr == 0] = 0.0
        acc = acc + a
    return c * acc


def _rotlet_grad_f64(t, src, L, eta):
    c = 1.0 / (8.0 * np.pi * eta)
    acc = np.zeros((len(t), 10))
    for s in range(len(src)):
        d = t - src[s]
        dr2 = ps.r2_kernel(d[:, 0], d[:, 1], d[:, 2])
        with np.errstate(divide="ignore", invalid="ignore"):
            D = np.where(dr2 < fr.EPS2, np.sqrt(fr.REG2 + dr2), np.sqrt(dr2))
            f3 = 1.0 / ((D * D) * D)
            hr = (3.0 * f3) / (D * D)
        l0, l1, l2 = L[s]
        m = [d[:, 2] * l1 - d[:, 1] * l2, d[:, 0] * l2 - d[:, 2] * l0, d[:, 1] * l0 - d[:, 0] * l1]
        e = [0.0, -l2, l1, l2, 0.0, -l0, -l1, l0, 0.0]
        a = np.zeros((len(t), 10))
        for i in range(3):
            for j in range(3):
                a[:, 3 * i + j] = f3 * e[3 * i + j] - (hr * m[i]) * d[:, j]
        a[dr2 == 0] = 0.0
        acc = acc + a
    return c * acc


def test_the_aux_kernels_in_float64_meet_k():
    fib, shell, body, (pts, pf, ptq), r = edge_case(5)
    worst = {}
    for eta in (0.37, 2.5):
        for name, got, ref in (("Oseen", _oseen_grad_f64(r, pts, pf, eta), gr.oseen_grad(r, pts, pf, eta)),
                               ("rotlet, points", _rotlet_grad_f64(r, pts, ptq, eta),
                                gr.rotlet_grad(r, pts, ptq, eta)),
                               ("rotlet, centres", _rotlet_grad_f64(r, body["centers"], body["torques"], eta),
                                gr.rotlet_grad(r, body["centers"], body["torques"], eta))):
            ext, S, K = ref
            q = gr.ratio(got, ext, S) / K[:, None]
            assert (q <= 1).all(), (name, q.max())
            worst[name] = max(worst.get(name, 0.0), float(q.max()))
    print("\nfloat64 aux kernels, worst ratio / K:", {k: f"{v:.3g}" for k, v in worst.items()})


# ---- the regularised branches are the derivative of the regularised velocities -------------------------------------
@pytest.mark.parametrize("which", ["oseen", "rotlet"])
def test_the_regularised_branch_is_the_derivative_of_the_oracle_velocity(which):
    rng = RNG(6)
    eta = 0.7
    src = rng.uniform(-1, 1, (1, 3))
    f = rng.normal(size=(1, 3))
    r = inside_eps(rng, src, 40)
    if which == "oseen":
        vel, grad = (lambda x: orc.oseen_contract(src, x, f, eta)), gr.oseen_grad(r, src, f, eta)
    else:
        vel, grad = (lambda x: orc.rotlet(src, x, f, eta)), gr.rotlet_grad(r, src, f, eta)
    G = np.asarray(grad[0][:, :9], dtype=np.float64).reshape(-1, 3, 3)
    h = 1e-9
    fd = np.zeros_like(G)
    for j in range(3):
        e = np.zeros(3)
        e[j] = h
        fd[:, :, j] = np.asarray((vel(r + e).astype(np.longdouble) - vel(r - e)) / (2 * np.longdouble(h)),
                                 dtype=np.float64)
        dist = np.linalg.norm(np.concatenate([r + e, r - e]) - src, axis=1)
        assert (dist < 9.1e-6).all() and (dist > 0).all()
    scale = np.abs(G).reshape(len(r), 9).max(axis=1)
    err = np.abs(G - fd).reshape(len(r), 9).max(axis=1) / scale
    print(f"\n{which}: regularised gradient vs central differences, worst {err.max():.3g} of the row's largest entry")
    assert (err <= 1e-4).all(), err.max()
    # the check sees a wrong factor of D: 3 r_i r_j (r.f) / (D^3 r^2) is of the size of the other terms, not r^2 / D^2
    # smaller
    if which == "oseen":
        bad = np.asarray(gr.oseen_grad(r, src, f, eta, defect="oseen_r_for_D")[0][:, :9], dtype=np.float64)
        bad_err = np.abs(bad.reshape(-1, 3, 3) - fd).reshape(len(r), 9).max(axis=1) / scale
        assert bad_err.max() > 1e2 * err.max(), (bad_err.max(), err.max())


# ---- sharp ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def case():
    return edge_case(7)


def test_the_edge_case_reaches_every_branch(case):
    fib, shell, body, points, r = case
    rows = branch_rows(r, fib, shell, body, points[0])
    missing = [k for k, v in rows.items() if not v.any()]
    assert not missing, missing


def _miss(case, defect, eta=0.37):
    fib, shell, body, points, r = case
    ext, S, K = gr.frame(fib, shell, body, r, eta, points, BG)
    bad, _, _ = gr.frame(fib, shell, body, r, eta, points, BG, defect=defect)
    with np.errstate(over="ignore", invalid="ignore"):
        q = gr.ratio(np.asarray(bad, dtype=np.float64), ext, S) / K[:, None]
    return np.nan_to_num(q, nan=np.inf).max(axis=1)


# defects only the row exactly at an eps edge can see, and the branch row that holds it
EDGE_ONLY = {"oseen_eps_strict": "Oseen, points: float64 r == EPS",
             "rotlet_eps_le": "rotlet, points: float64 r^2 == EPS2"}


@pytest.mark.parametrize("defect", gr.DEFECTS)
def test_each_planted_defect_misses_its_bound(case, defect):
    miss = _miss(case, defect)
    print(f"\n{defect}: misses its bound by {miss.max():.3g} K")
    assert miss.max() > MISS, (defect, miss.max())
    if defect in EDGE_ONLY:
        fib, shell, body, points, r = case
        at_edge = branch_rows(r, fib, shell, body, points[0])[EDGE_ONLY[defect]]
        assert at_edge.any() and (miss[at_edge] > MISS).any()


def test_the_good_restatement_is_its_own_bound(case):
    """ext rounded to float64 meets the bound with room: the rows are finite and K u S is not degenerate"""
    fib, shell, body, points, r = case
    ext, S, K = gr.frame(fib, shell, body, r, 2.5, points, BG)
    assert np.isfinite(np.asarray(ext, dtype=np.float64)).all() and (K > 0).all()
    assert (gr.ratio(np.asarray(ext, dtype=np.float64), ext, S) <= 1).all()


def test_interior_rows_hold_the_last_bodys_rigid_gradient():
    _, _, body, _, _ = edge_case(8)
    kind, radii = np.array([1, 1, 2]), np.array([[0.4, 0, 0], [0.4, 0, 0], [0.5, 0.3, 0.35]])
    uw = RNG(3).uniform(-0.5, 0.5, (3, 6))
    r = body["centers"][1] + RNG(4).uniform(-0.3, 0.3, (200, 3))
    mask, rigid = gr.interior(r, body, kind, radii, uw)
    in2 = gr.interior(r, dict(centers=body["centers"][2:]), kind[2:], radii[2:], uw[2:])[0]
    assert mask.any() and in2.any() and (mask & ~in2).any()
    assert np.array_equal(rigid[in2], np.broadcast_to(gr.rigid_gradient(uw[2, 3:]), (in2.sum(), 10)), equal_nan=True)
    assert np.isnan(rigid[mask, 9]).all()

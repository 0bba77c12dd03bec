"""CPU tests of the entry-wise criterion of tests/body_block_reference.py, which tests/test_gpu_system_ext.py applies to
the body block, the fiber-body links and the body preconditioner on the device: |dev - ext| <= K u S per entry, ext the
restatement in np.longdouble, S the same computation on absolute values, K fixed in advance from the kernels' summation
depth (the module's docstring derives each).

The criterion is attainable: the float64 restatement, summing in the kernels' order, meets every bound on the shapes of
the GPU tests (bodies of 1 .. 2000 nodes, 40 bodies in one flow and one with no fiber bound, fibers of 8 .. 128 nodes
with free fibers before bound ones and 60 fibers on one body, nucleation sites at |s| = 1e-6 .. 1e2, node weights over
1e-3 .. 1e3).  It is sharp: every planted defect misses its bound by at least DEFECT_FACTOR x K on some entry."""
import numpy as np
import pytest

import body_block_reference as bb
import system_reference as sr
from oracle.fiber_fd import compute_matrices

BODY_NODES = (1, 2, 85, 255, 256, 257, 511, 513, 2000)
FIBER_NODES = (8, 31, 32, 33, 64, 96, 128)
ETA = 0.9
# the smallest factor by which a defect must miss its bound (ratio / K); every defect below misses by far more
DEFECT_FACTOR = 1e10


def body_case(seed, body_nodes=BODY_NODES, n_bodies=40, fiber_nodes=FIBER_NODES, n_free=6, on_first=60, real=False):
    """n_bodies bodies (the first len(body_nodes) of the given sizes, the others of 3 .. 40 nodes) on spheres of radius 0.4
    around centres 1.5 apart or more; n_free free fibers, then on_first fibers bound to body 0, then one or two per body
    up to the last, to which none is bound.  Node weights 10^U(-3, 3); ex / ey / ez random stand-ins.  real=True: the
    reference's D_2_0 / D_3_0 (compute_matrices), else random ones.  Returns (fib, ops, links, bodies)."""
    rng = np.random.default_rng(seed)
    sizes = list(body_nodes) + [int(k) for k in rng.integers(3, 41, n_bodies - len(body_nodes))]
    g = np.stack(np.meshgrid(*[np.arange(4)] * 3, indexing="ij"), axis=-1).reshape(-1, 3)[:n_bodies]
    centers = 1.6 * g + rng.uniform(-0.05, 0.05, (n_bodies, 3)) - 2.4
    pos, nrm = [], []
    for c, n in zip(centers, sizes):
        e = rng.normal(size=(n, 3))
        e /= np.linalg.norm(e, axis=1)[:, None]
        pos.append(c + 0.4 * e), nrm.append(e)
    pos, nrm = np.concatenate(pos), np.concatenate(nrm)
    nb = pos.shape[0]
    bodies = dict(pos=pos, normals=nrm, centers=centers, n_nodes=sizes, weights=10.0 ** rng.uniform(-3, 3, nb),
                  ex=rng.normal(size=(nb, 3)), ey=rng.normal(size=(nb, 3)), ez=rng.normal(size=(nb, 3)))
    body_of = [-1] * n_free + [0] * on_first
    for b in range(1, n_bodies - 1):
        body_of += [b] * (1 + b % 2)
    nfib = len(body_of)
    n_nodes = [fiber_nodes[i % len(fiber_nodes)] for i in range(nfib)]
    lengths = rng.uniform(0.5, 2.0, nfib)
    fpos, xs = [], []
    for n, L in zip(n_nodes, lengths):
        t = rng.normal(size=3)
        t /= np.linalg.norm(t)
        fpos.append(rng.uniform(-3.5, 3.5, 3) + np.linspace(0, L, n)[:, None] * t)
        x = rng.normal(size=(n, 3))
        xs.append(x / np.linalg.norm(x, axis=1)[:, None])
    fib = dict(pos=np.concatenate(fpos), n_nodes=n_nodes, lengths=list(lengths))
    nset = sorted(set(n_nodes))
    if real:
        mats = {n: compute_matrices(n) for n in nset}
        D2, D3 = {n: mats[n]["D_2_0"] for n in nset}, {n: mats[n]["D_3_0"] for n in nset}
    else:
        D2, D3 = ({n: rng.normal(size=(n, n)) for n in nset} for _ in range(2))
    ops = dict(xs=np.concatenate(xs), D_2_0=D2, D_3_0=D3,
               length_prev=list(lengths * (1 + rng.choice([-1, 1], nfib) * rng.uniform(0.02, 0.1, nfib))))
    s = rng.normal(size=(nfib, 3))
    s *= (10.0 ** rng.uniform(-6, 2, nfib) / np.linalg.norm(s, axis=1))[:, None]
    site = np.array([centers[b] + s[i] if b >= 0 else rng.normal(size=3) for i, b in enumerate(body_of)])
    links = dict(body=np.array(body_of), site=site, rigidity=rng.uniform(0.5, 2.0, nfib))
    return fib, ops, links, bodies


def body_x(rng, bodies, densities=True, motion=True):
    """x_bodies: node densities (or zeros), then U and omega of each body (or zeros)"""
    out = []
    for n in bodies["n_nodes"]:
        d = rng.normal(size=3 * n) if densities else np.zeros(3 * n)
        out += [d, rng.normal(size=6) if motion else np.zeros(6)]
    return np.concatenate(out)


def bound_stats(links, fib, n_bodies):
    """per body: (largest node count, number) of its bound fibers"""
    out = []
    for b in range(n_bodies):
        ns = [int(n) for n, bb_ in zip(fib["n_nodes"], links["body"]) if bb_ == b]
        out.append((max(ns) if ns else 0, len(ns)))
    return out


def k_ft_per_body(links, fib, n_bodies):
    return np.array([bb.k_ft(n, m) for n, m in bound_stats(links, fib, n_bodies)])


@pytest.fixture(scope="module")
def case():
    fib, ops, links, bodies = body_case(5)
    rng = np.random.default_rng(6)
    x_f = rng.normal(size=4 * fib["pos"].shape[0])
    x_b = body_x(rng, bodies)
    return fib, ops, links, bodies, x_f, x_b


def link_refs(fib, ops, links, bodies, x_f, x_b, **kw):
    return [bb.link_terms(fib, ops, links, bodies, x_f, x_b, dtype=d, absolute=a, **kw)
            for d, a in ((np.float64, False), (np.longdouble, False), (np.longdouble, True))]


def test_float64_link_terms_meet_their_bounds_and_agree_with_the_restatement(case):
    assert np.finfo(np.longdouble).nmant >= 63
    fib, ops, links, bodies, x_f, x_b = case
    (l64, _, ft64), (le, _, fte), (ls, _, fts) = link_refs(fib, ops, links, bodies, x_f, x_b)
    worst_l = bb.ratio(l64, le, ls).max()
    kft = k_ft_per_body(links, fib, len(bodies["n_nodes"]))
    r_ft = bb.ratio(ft64, fte, fts)
    assert worst_l <= bb.K_LINK_ROWS and (r_ft <= kft[:, None]).all(), (worst_l, r_ft.max())
    # the last body has no bound fiber: its sums are exact zeros; free fibers' link rows too
    assert np.all(ft64[-1] == 0) and np.all(l64[np.asarray(links["body"]) < 0] == 0)
    # the same quantities as tests/system_reference.py states them (the GPU tests' norm gate)
    vel, ft = sr.link_conditions(fib, ops, links, bodies, x_f, x_b)
    assert np.abs(vel - l64).max() <= 1e-13 * np.abs(vel).max()
    assert np.abs(ft - ft64).max() <= 1e-12 * np.abs(ft).max()
    print(f"\nfloat64 link rows: worst |d|/(u S) {worst_l:.2f} (K {bb.K_LINK_ROWS}); "
          f"forces / torques {(r_ft / kft[:, None]).max():.3f} of K")


@pytest.mark.parametrize("real", [False, True])
def test_float64_centre_flow_meets_its_bound(real):
    fib, ops, links, bodies = body_case(7, real=real)
    rng = np.random.default_rng(8)
    x_f, x_b = rng.normal(size=4 * fib["pos"].shape[0]), body_x(rng, bodies)
    (_, _, ft64), (_, _, fte), (_, _, fts) = link_refs(fib, ops, links, bodies, x_f, x_b)
    trg = np.concatenate([bodies["pos"], fib["pos"][np.concatenate([[0], np.cumsum(fib["n_nodes"])[:-1]])]])
    c = bodies["centers"]
    v64 = bb.centre_flow(trg, c, ft64[:, :3], ft64[:, 3:], ETA, dtype=np.float64)
    ve = bb.centre_flow(trg, c, fte[:, :3], fte[:, 3:], ETA)
    vs = bb.centre_flow(trg, c, fts[:, :3], fts[:, 3:], ETA, absolute=True)
    K = bb.k_flow(len(c)) + k_ft_per_body(links, fib, len(c)).max()
    r = bb.ratio(v64, ve, vs)
    assert r.max() <= K, (r.max(), K)
    print(f"\nfloat64 centre flow: worst |d|/(u S) {r.max():.2f} (K {K})")


def test_float64_body_rows_meet_their_bounds(case):
    _, _, _, bodies, _, x_b = case
    v = np.random.default_rng(9).normal(size=bodies["pos"].shape)
    r = bb.ratio(bb.body_rows(bodies, v, x_b, dtype=np.float64), *bb.ext_and_scale(bb.body_rows, bodies, v, x_b))
    worst_node, worst_kt = 0.0, 0.0
    off = 0
    for n in bodies["n_nodes"]:
        worst_node = max(worst_node, r[off:off + 3 * n].max(initial=0.0))
        worst_kt = max(worst_kt, r[off + 3 * n:off + 3 * n + 6].max() / bb.k_kt(n))
        off += 3 * n + 6
    assert worst_node <= bb.K_NODE and worst_kt <= 1.0, (worst_node, worst_kt)
    ref = sr.body_matvec(bodies, v, x_b)
    assert np.abs(bb.body_rows(bodies, v, x_b, dtype=np.float64) - ref).max() <= 1e-13 * np.abs(ref).max()
    print(f"\nfloat64 body rows: node rows {worst_node:.2f} (K {bb.K_NODE}), K^T lambda rows {worst_kt:.3f} of K")


def gemv_case(seed, m):
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(m, m)) * 10.0 ** rng.uniform(-3, 3, m)[None, :]
    return A, rng.normal(size=m)


@pytest.mark.parametrize("n", [1, 2, 85, 255, 257, 513])
def test_float64_gemv_meets_its_bound(n):
    m = 3 * n + 6
    A, x = gemv_case(n, m)
    r = bb.ratio(bb.gemv_rows(A, x, dtype=np.float64), *bb.ext_and_scale(bb.gemv_rows, A, x))
    assert r.max() <= bb.k_gemv(m), (r.max(), bb.k_gemv(m))
    print(f"\nfloat64 GEMV, m = {m}: worst |d|/(u S) {r.max():.2f} (K {bb.k_gemv(m)})")


def _worst_over_k(r, K):
    return float(np.max(r / K))


@pytest.mark.parametrize("defect", bb.LINK_DEFECTS)
def test_link_criterion_catches_planted_defects(case, defect):
    fib, ops, links, bodies, x_f, x_b = case
    _, (le, _, fte), (ls, _, fts) = link_refs(fib, ops, links, bodies, x_f, x_b)
    bad, _, ft_bad = bb.link_terms(fib, ops, links, bodies, x_f, x_b, dtype=np.float64, defect=defect)
    if defect == "omega_site_sign":
        f = _worst_over_k(bb.ratio(bad, le, ls), bb.K_LINK_ROWS)
    else:
        f = _worst_over_k(bb.ratio(ft_bad, fte, fts), k_ft_per_body(links, fib, len(bodies["n_nodes"]))[:, None])
    print(f"\n{defect}: misses its bound by {f:.3g} x K")
    assert f > DEFECT_FACTOR, (defect, f)


@pytest.mark.parametrize("defect", bb.BODY_DEFECTS)
def test_body_criterion_catches_planted_defects(case, defect):
    _, _, _, bodies, _, x_b = case
    v = np.random.default_rng(9).normal(size=bodies["pos"].shape)
    ext, S = bb.ext_and_scale(bb.body_rows, bodies, v, x_b)
    r = bb.ratio(bb.body_rows(bodies, v, x_b, dtype=np.float64, defect=defect), ext, S)
    K = np.empty_like(r)
    off = 0
    for n in bodies["n_nodes"]:
        K[off:off + 3 * n] = bb.K_NODE
        K[off + 3 * n:off + 3 * n + 6] = bb.k_kt(n)
        off += 3 * n + 6
    f = _worst_over_k(r, K)
    print(f"\n{defect}: misses its bound by {f:.3g} x K")
    assert f > DEFECT_FACTOR, (defect, f)


def test_gemv_criterion_catches_a_shifted_row_block():
    m = 3 * 85 + 6
    A, x = gemv_case(85, m)
    f = _worst_over_k(bb.ratio(bb.gemv_rows(A, x, dtype=np.float64, defect="shift_block_32"),
                               *bb.ext_and_scale(bb.gemv_rows, A, x)), bb.k_gemv(m))
    print(f"\nshift_block_32: misses its bound by {f:.3g} x K")
    assert f > DEFECT_FACTOR, f


def test_lane_sum_follows_the_kernels_order():
    # a sum whose value depends on the order: lanes first, then the tree / the slices in turn
    t = np.array([1.0, 2.0 ** -53, 2.0 ** -53, -1.0] + [0.0] * 60)
    assert bb.lane_sum(t, 2) == ((1.0 + 2.0 ** -53) + 0.0) + (2.0 ** -53 + -1.0)
    assert bb.lane_sum(np.arange(20.0), 8, tree=False) == sum(np.arange(20.0))
    assert bb.lane_sum(np.ones(257), 256) == 257.0

"""The criterion of tests/flow_reference.py is attainable and sharp, without a GPU.

Attainable: the oracle's float64 restatement of the flows (FiberContainerFiniteDifference::flow with its self block,
Periphery::flow, BodyContainer::flow, the point sources, the background and System::apply_matvec's v_all) meets
|f64 - ext| <= K u S on every row of a system built to reach the kernels' edges: fiber nodes exactly EPS apart along an
axis (float64 r == EPS, the regularised side), one ulp beyond it, closer than EPS, coincident, nodes of different fibers
within EPS, targets on a point source, at EPS and one ulp either side of it, on a body centre and on the fiber nodes,
per-fiber forces over 1e-3 .. 1e3 and eta != 1.  The worst fraction of K it uses is below FRACTION (measured: 0.051 for
the fiber flow, 0.029 at targets and on the matvec's rows; the oracle sums in its own order and evaluates every
pair in its own instruction order, so it is a float64 evaluation as unlike the kernels as any).

Sharp: each planted defect of flow_reference.DEFECTS misses its bound on some row by more than MISS times K.
"""
import numpy as np
import pytest

import flow_reference as fr
import oracle as orc

FRACTION = 0.1
MISS = 1e6
ETA = 2.5


def _fiber(x, yz):
    x = np.asarray(x, dtype=np.float64)
    return np.stack([x, np.full_like(x, yz[0]), np.full_like(x, yz[1])], axis=1)


def edge_fibers(rng, nodes=(8, 16, 31), spread=3.0):
    """fibers at the self term's edges, then random straight fibers of the given node counts; per-fiber forces of
    magnitude 1e-3 .. 1e3"""
    eps = fr.EPS
    pos = [_fiber([0.0, eps, 0.3, 0.6, 0.9], (1.3, -0.7)),                      # r == EPS: regularised (<=)
           _fiber([0.0, np.nextafter(eps, 1.0), 0.5, 1.0], (0.5, 1.9)),         # one ulp beyond: not regularised
           _fiber([2.0, 2.0 + 4e-6, 2.4, 2.8, 3.2, 3.6], (-1.1, 0.4)),          # 0 < r < EPS
           _fiber([-1.0, -0.5, -0.5, 0.0], (-0.3, -2.2)),                       # coincident nodes: r == 0, skipped
           _fiber([0.0, 0.4, 0.8], (-2.0, 0.0)),                                # these two fibers' first nodes are
           _fiber([3e-6, 0.5, 1.0, 1.5], (-2.0, 0.0))]                          # 3e-6 apart
    lengths = [0.9, 1.0, 1.6, 1.0, 0.8, 1.5]
    for n in nodes:
        L = rng.uniform(0.5, 2.0)
        h = rng.normal(size=3)
        pos.append(rng.uniform(-spread, spread, 3) + np.linspace(0, L, n)[:, None] * (h / np.linalg.norm(h)))
        lengths.append(L)
    n_nodes = [len(p) for p in pos]
    scale = np.repeat(10.0 ** rng.uniform(-3, 3, len(pos)), n_nodes)
    forces = rng.normal(size=(sum(n_nodes), 3)) * scale[:, None]
    return dict(pos=np.concatenate(pos), n_nodes=n_nodes, lengths=lengths, forces=forces)


def shell_and_bodies(rng, n_shell=120, per=40, centers=((0.0, 1.5, -1.5), (1.0, -0.5, 2.0), (1.3, -0.5, 2.0))):
    d = rng.normal(size=(n_shell, 3))
    d /= np.linalg.norm(d, axis=1)[:, None]
    shell = dict(pos=d * np.array([7.8, 4.16, 4.16]), normals=-d, density=rng.uniform(-1, 1, (n_shell, 3)))
    centers = np.array(centers, dtype=np.float64)
    e = rng.normal(size=(len(centers) * per, 3))
    e /= np.linalg.norm(e, axis=1)[:, None]
    pos = np.repeat(centers, per, axis=0) + 0.4 * e
    body = dict(pos=pos, normals=e, density=rng.uniform(-1, 1, pos.shape), centers=centers,
                forces=rng.uniform(-1, 1, centers.shape), torques=rng.uniform(-1, 1, centers.shape))
    return shell, body


def edge_targets(rng, fib, body, pts, n_free=60):
    """free targets, the fiber nodes, a target on a point source and at +-EPS and one ulp either side along x from
    points and body centres whose x is 0 (so that dy = dz = 0 exactly), and the body centres"""
    eps = fr.EPS
    deltas = [np.nextafter(eps, 0.0), eps, np.nextafter(eps, 1.0), 4e-6]
    out = [rng.uniform(-2.5, 2.5, (n_free, 3)), fib["pos"], pts[:1], body["centers"]]
    for p in list(pts[:2]) + [body["centers"][0]]:
        assert p[0] == 0.0
        out += [p + [[s * dl, 0, 0] for dl in deltas for s in (1, -1)]]
    return np.concatenate(out)


def point_sources(rng):
    pts = np.array([[0.0, 0.7, -0.4], [0.0, -0.9, 1.2], [0.35, 0.1, 0.2]])
    return pts, rng.normal(size=(3, 3)), rng.normal(size=(3, 3))


BG = ([1, 0, 2], np.array([0.5, -0.25, 0.125]), np.array([0.1, 0.0, -0.3]))


@pytest.fixture(scope="module")
def case():
    rng = np.random.default_rng(2024)
    fib = edge_fibers(rng)
    shell, body = shell_and_bodies(rng)
    points = point_sources(rng)
    r = edge_targets(rng, fib, body, points[0])
    return fib, shell, body, points, r


def _worst(got, ref):
    ext, S, K = ref
    return float((fr.ratio(got, ext, S) / np.asarray(K)[:, None]).max())


def _f64_at_targets(fib, shell, body, points, r):
    v = orc.fiber_flow(r, fib["pos"], fib["n_nodes"], fib["lengths"], fib["forces"], ETA, subtract_self=False)
    v += orc.periphery_flow(r, shell["pos"], shell["normals"], shell["density"], ETA)
    v += orc.body_flow(r, body["pos"], body["normals"], body["density"], body["centers"], body["forces"],
                       body["torques"], ETA)
    pts, pf, ptq = points
    v += orc.oseen_contract(pts, r, pf, ETA) + orc.rotlet(pts, r, ptq, ETA)
    return v + BG[2][None, :] + r[:, BG[0]] * BG[1][None, :]


def _f64_fiber_flow(fib, r, subtract_self):
    return orc.fiber_flow(r, fib["pos"], fib["n_nodes"], fib["lengths"], fib["forces"], ETA, subtract_self)


def _ranges(fib, shell, body):
    nfib = len(fib["n_nodes"])
    return (2, nfib - 1, 10, len(shell["pos"]) - 7, 5, len(body["pos"]) - 3)


def _window_rows(fib, shell, body, v, ranges):
    fa, fb, sa, sb, ba, bb = fr.window(fib, shell, body, ranges)
    nf, ns = len(fib["pos"]), len(shell["pos"])
    return np.concatenate([v[fa:fb], v[nf + sa:nf + sb], v[nf + ns + ba:nf + ns + bb]])


def test_the_float64_evaluation_meets_the_bound(case):
    fib, shell, body, points, r = case
    worst = {
        "velocity_at_targets": _worst(_f64_at_targets(fib, shell, body, points, r),
                                      fr.velocity_at_targets(fib, shell, body, r, ETA, points, BG)),
        "fiber_flow": _worst(_f64_fiber_flow(fib, r, False), fr.fiber_flow(fib, r, ETA)),
        "fiber_flow subtract_self": _worst(_f64_fiber_flow(fib, r, True), fr.fiber_flow(fib, r, ETA, True)),
    }
    v = orc.matvec_flow(fib, shell, body, ETA)
    worst["matvec"] = _worst(v, fr.matvec(fib, shell, body, ETA))
    rg = _ranges(fib, shell, body)
    worst["matvec window"] = _worst(_window_rows(fib, shell, body, v, rg), fr.matvec(fib, shell, body, ETA, rg))
    print("\nworst ratio / K of the float64 evaluation:", {k: f"{w:.3g}" for k, w in worst.items()})
    assert max(worst.values()) < FRACTION, worst


def test_the_self_term_does_not_cancel_within_eps(case):
    """within EPS the pair sum holds the unregularised pair and the self term subtracts the regularised one: the fiber
    rows there are dominated by the leftover, and the pair at float64 r == EPS sits on the regularised side"""
    fib, _, _, _, _ = case
    n0 = fib["pos"][:3]
    sub, _, _ = fr.fiber_flow(fib, n0, ETA, True)
    pairs_only, _, _ = fr.fiber_flow(fib, n0, ETA, False)
    strict, _, _ = fr.fiber_flow(fib, n0, ETA, True, defect="self_eps_strict")
    assert np.all(np.abs(sub[:2] - pairs_only[:2]) > 0)
    assert np.all(np.abs(strict[:2] - sub[:2]) > 1e-3 * np.abs(sub[:2]))   # r == EPS decides the branch


def _defect_miss(case, defect):
    fib, shell, body, points, r = case
    if defect in ("self_j_short", "self_no_reg", "self_eps_strict", "weights_not_halved"):
        return _worst(_f64_fiber_flow(fib, r, True), fr.fiber_flow(fib, r, ETA, True, defect=defect))
    if defect in ("rotlet_eps_le", "point_r0_kept", "bg_component", "periphery_no_eta"):
        return _worst(_f64_at_targets(fib, shell, body, points, r),
                      fr.velocity_at_targets(fib, shell, body, r, ETA, points, BG, defect=defect))
    v = orc.matvec_flow(fib, shell, body, ETA)
    rg = _ranges(fib, shell, body)
    return _worst(_window_rows(fib, shell, body, v, rg), fr.matvec(fib, shell, body, ETA, rg, defect=defect))


@pytest.mark.parametrize("defect", [d for d in fr.DEFECTS if d != "interior_first_wins"])
def test_each_planted_defect_misses_its_bound(case, defect):
    miss = _defect_miss(case, defect)
    print(f"\n{defect}: worst ratio / K {miss:.3g}")
    assert miss > MISS, (defect, miss)


def test_interior_first_wins_changes_overlapping_rows(case):
    """bodies 1 and 2 overlap; rows inside both take body 2's rigid motion, bitwise"""
    _, _, body, _, _ = case
    rng = np.random.default_rng(3)
    kind, radii = np.array([1, 1, 2]), np.array([[0.4, 0, 0], [0.4, 0, 0], [0.5, 0.3, 0.35]])
    uw = rng.uniform(-0.5, 0.5, (3, 6))
    r = np.concatenate([body["centers"][1] + rng.uniform(-0.3, 0.3, (200, 3)), rng.uniform(-2, 2, (50, 3))])
    m, v = fr.interior(r, body, kind, radii, uw)
    m1, v1 = fr.interior(r, body, kind, radii, uw, defect="interior_first_wins")
    assert np.array_equal(m, m1) and m.sum() > 20
    assert not np.array_equal(v[m], v1[m])
    both = fr.interior(r, dict(centers=body["centers"][2:]), kind[2:], radii[2:], uw[2:])[0] & \
        fr.interior(r, dict(centers=body["centers"][1:2]), kind[1:2], radii[1:2], uw[1:2])[0]
    assert both.any() and np.array_equal(v[both], fr.interior(r[both], dict(centers=body["centers"][2:]), kind[2:],
                                                              radii[2:], uw[2:])[1])

"""skb_flow_listener_gradient held output by output to the long-double restatement of tests/gradient_reference.py:
|dev - ext| <= K u S for each of the 9 gradient entries and the pressure of every row, K fixed from the kernel source
before any GPU run (the module's docstring derives it).  Every body's interior kind is 0 for the edge rows, so each row
is a fluid point.  Every call runs twice and the two results are bitwise equal.

Rows: on fiber, shell and body nodes, point sources and body centres (r == 0); at subnormal-r^2 offsets from a fiber
node; at the last float64 offset each eps rule still regularises and one ulp beyond, for the Oseen rule around a point
source and the rotlet rule around a point source and a body centre; strictly inside eps; far (|r| from 1e3 to 1e6) from
force-free source sets.  Plan shapes: n_trg in {1, 2, 3, 255, 257, 4099} (the gradient kinds run two targets per
thread), source counts with a ragged last 128-tile, a periphery of about 20 000 nodes against a few targets (several
source splits).  eta 0.37 and 2.5, per-fiber forces from 1e-3 to 1e3.  The test asserts that each branch it claims
was reached.

Independent of the restatement, the device gradient is the central difference of the device's own velocity_field, with
both points in one branch: inside eps of a point source (h = 1e-9) and away from every source (h = 1e-5).  And
set_self_exclusion(True) leaves it bitwise unchanged (Evaluator::gradient passes no fiber ids).

Worst ratio / K, gradient / pressure (test_worst_ratios_report prints them), on an H100 80GB HBM3 at 700 W:
    each part alone on the edge rows:
        Stokeslet: fibers                        0.0264 / 0.0168
        stresslet: periphery                     0.0178 / 0.0142
        bodies: surface, centre forces, torques  0.0173 / 0.0083
        Oseen: point forces                      0.093 / 0.0588
        rotlet: point torques                    0.134 / 0 (no pressure)
        background                               0 / 0 (exact)
    whole frames:
        edge rows                                0.0308 / 0.0118
        plan shapes                              0.0358 / 0.0173
        far rows, force-free                     0.00271 / 0.00186
        large periphery                          8.41e-05 / 5.67e-05
    central differences (relative), inside eps / away from sources: 2.83e-08 / 3.43e-10
"""
import numpy as np
import pytest

import gradient_reference as gr
import pair_sum_reference as ps
import skellysim_b200 as skb
from skellysim_b200 import capi
from test_flow_ext_cpu import BG, edge_fibers, shell_and_bodies
from test_gpu_flow import ft_of, load
from test_listener_gradient_ext_cpu import branch_rows, edge_case, inside_eps

pytestmark = pytest.mark.gpu
WORST = {}


def _set_frame(fl, fib, shell, body, eta):
    nb = len(body["centers"])
    fl.set_listener_frame(fib["forces"], shell["density"], body["density"], ft_of(body), np.zeros((nb, 6)),
                          np.zeros(nb, dtype=np.int32), np.full((nb, 3), 0.4), eta)


def _open(fib, shell, body, points, bg, eta):
    fl = skb.Flow(0)
    load(fl, fib, shell, body)
    if points is not None:
        fl.set_point_sources(*points)
    if bg is not None:
        fl.set_background(*bg)
    _set_frame(fl, fib, shell, body, eta)
    return fl


def _gradient(fl, r):
    """(n, 10) of capi.listener_gradient, asserted bitwise equal over two calls"""
    a = capi.listener_gradient(fl, r)
    b = capi.listener_gradient(fl, r)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1], equal_nan=True)
    return np.concatenate([a[0].reshape(len(r), 9), a[1][:, None]], axis=1)


def _check(name, dev, ref):
    ext, S, K = ref
    assert np.isfinite(dev).all(), name
    q = gr.ratio(dev, ext, S) / np.asarray(K, dtype=np.float64)[:, None]
    parts = {"gradient": q[:, :9], "pressure": q[:, 9]}
    for k, v in parts.items():
        WORST[f"{name}, {k}"] = max(WORST.get(f"{name}, {k}", 0.0), float(v.max()) if v.size else 0.0)
    bad = np.argwhere(q > 1)
    assert bad.size == 0, (name, bad[:5].tolist(), float(q.max()))


@pytest.mark.parametrize("eta", [0.37, 2.5])
def test_edge_rows(eta):
    fib, shell, body, points, r = edge_case(11)
    rows = branch_rows(r, fib, shell, body, points[0])
    missing = [k for k, v in rows.items() if not v.any()]
    assert not missing, missing
    with _open(fib, shell, body, points, BG, eta) as fl:
        dev = _gradient(fl, r)
    _check("edge rows", dev, gr.frame(fib, shell, body, r, eta, points, BG))


_E3 = np.zeros((0, 3))
_NO_FIB = dict(pos=_E3, n_nodes=[], lengths=[], forces=_E3)
_NO_SHELL = dict(pos=_E3, normals=_E3, density=_E3)
_NO_BODY = dict(pos=_E3, normals=_E3, density=_E3, centers=_E3, forces=_E3, torques=_E3)
PARTS = ("Stokeslet: fibers", "stresslet: periphery", "bodies: surface, centre forces and torques",
         "Oseen: point forces", "rotlet: point torques", "background")


@pytest.mark.parametrize("part", PARTS)
def test_each_part_alone_on_the_edge_rows(part):
    """one source class at a time (the others empty, or the point sources' forces or torques zero), so that the worst
    ratio of each part is its own"""
    fib, shell, body, (pts, pf, ptq), r = edge_case(17)
    z = np.zeros_like(pf)
    fib_, shell_, body_, points, bg = _NO_FIB, _NO_SHELL, _NO_BODY, None, None
    if part.startswith("Stokeslet"):
        fib_ = fib
    elif part.startswith("stresslet"):
        shell_ = shell
    elif part.startswith("bodies"):
        body_ = body
    elif part.startswith("Oseen"):
        points = (pts, pf, z)
    elif part.startswith("rotlet"):
        points = (pts, z, ptq)
    else:
        bg = BG
    eta = 0.37
    with _open(fib_, shell_, body_, points, bg, eta) as fl:
        dev = _gradient(fl, r)
    _check(part, dev, gr.frame(fib_, shell_, body_, r, eta, points, bg))


def _force_free(fib):
    """per-fiber forces whose trapezoid-weighted sum vanishes (to rounding)"""
    f = fib["forces"].copy()
    w = ps.trapezoid_weights(fib["n_nodes"], fib["lengths"])
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
    for a, b in zip(off[:-1], off[1:]):
        f[a:b] -= (w[a:b, None] * f[a:b]).sum(axis=0) / w[a:b].sum()
    return dict(fib, forces=f)


def test_far_rows_of_force_free_sources():
    rng = np.random.default_rng(12)
    fib = _force_free(edge_fibers(rng, (8, 16, 31)))
    shell, body = shell_and_bodies(rng, 200, 40)
    body = dict(body, forces=np.zeros_like(body["forces"]))
    u = rng.normal(size=(300, 3))
    r = u / np.linalg.norm(u, axis=1)[:, None] * 10.0 ** rng.uniform(3, 6, (300, 1))
    eta = 0.37
    with _open(fib, shell, body, None, None, eta) as fl:
        dev = _gradient(fl, r)
    _check("far rows, force-free", dev, gr.frame(fib, shell, body, r, eta))


SHAPES = {
    # n_fibers of each size, n_shell, per-body nodes
    "ragged": ((8, 16, 31, 64, 129), 333, 43),
    "tile multiples": ((64, 64), 256, 64),
}


@pytest.mark.parametrize("n_trg", [1, 2, 3, 255, 257, 4099])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_plan_shapes(shape, n_trg):
    nodes, n_shell, per = SHAPES[shape]
    fib, shell, body, points, edge = edge_case(13, nodes, n_shell, per, n_free=0)
    rng = np.random.default_rng(n_trg)
    pool = np.concatenate([edge, rng.uniform(-3, 3, (n_trg, 3))])
    r = pool[rng.permutation(len(pool))[:n_trg]]
    eta = 2.5
    with _open(fib, shell, body, points, BG, eta) as fl:
        dev = _gradient(fl, r)
    _check("plan shapes", dev, gr.frame(fib, shell, body, r, eta, points, BG))


def test_a_large_periphery_against_few_targets():
    """about 20 000 periphery nodes, 7 targets (one on a node): the planner splits the sources many ways"""
    rng = np.random.default_rng(14)
    fib = edge_fibers(rng, (8,))
    shell, body = shell_and_bodies(rng, 20011, 40)
    r = np.concatenate([shell["pos"][:1], shell["pos"][-1:] * 0.999, rng.uniform(-2, 2, (5, 3))])
    eta = 0.37
    with _open(fib, shell, body, None, BG, eta) as fl:
        dev = _gradient(fl, r)
    _check("large periphery", dev, gr.frame(fib, shell, body, r, eta, None, BG))


# ---- independent of the restatement --------------------------------------------------------------------------------
def _fd(fl, r, h):
    G = np.zeros((len(r), 3, 3))
    for j in range(3):
        e = np.zeros(3)
        e[j] = h
        G[:, :, j] = (fl.velocity_field(r + e).astype(np.longdouble) - fl.velocity_field(r - e)) / \
            (2 * np.longdouble(h))
    return G


def test_the_gradient_is_the_derivative_of_the_device_velocity():
    fib, shell, body, points, _ = edge_case(15)
    rng = np.random.default_rng(15)
    pts = points[0]
    near = inside_eps(rng, pts, 20)
    nodes = np.concatenate([fib["pos"], shell["pos"], body["pos"], pts, body["centers"]])
    far = rng.uniform(-2.5, 2.5, (4000, 3))
    far = far[np.linalg.norm(far[:, None, :] - nodes[None], axis=2).min(axis=1) > 0.3][:60]
    assert len(far) >= 30
    eta = 0.37
    with _open(fib, shell, body, points, BG, eta) as fl:
        for name, r, h, rel in (("inside eps of a point source", near, 1e-9, 1e-4), ("away from sources", far, 1e-5,
                                                                                     1e-6)):
            G = _gradient(fl, r)[:, :9].reshape(-1, 3, 3)
            fd = _fd(fl, r, h)
            scale = np.abs(G).reshape(len(r), 9).max(axis=1)
            err = np.abs(G - fd).reshape(len(r), 9).max(axis=1) / scale
            WORST[f"central differences, {name} (relative)"] = float(err.max())
            assert (err <= rel).all(), (name, err.max())


def test_self_exclusion_leaves_the_gradient_unchanged():
    fib, shell, body, points, r = edge_case(16)
    with _open(fib, shell, body, points, BG, 0.37) as fl:
        a = _gradient(fl, r)
        fl.set_self_exclusion(True)
        _set_frame(fl, fib, shell, body, 0.37)
        b = _gradient(fl, r)
    assert np.array_equal(a, b)


def test_worst_ratios_report():
    print("\nworst ratio / K:")
    for k, v in sorted(WORST.items()):
        print(f"    {k:52s} {v:.3g}")

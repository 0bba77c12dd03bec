"""CPU tests of the entry-wise criterion of tests/fiber_gemv_reference.py, which tests/test_gpu_fiber_gemv_ext.py applies
to fiber_gemv_kernel<MODE> on the device: |dev - ext| <= K u S per entry, ext the restatement in np.longdouble, S the
same computation on absolute values, K fixed in advance from the kernel's summation depth (the module's docstring
derives each).

The criterion is attainable: the float64 restatement, summing in the kernel's order, meets every bound on the shapes of
the GPU tests -- fibers of 4 .. 128 nodes with small and large ones alternating, x and v scaled per fiber over
1e-3 .. 1e3, length_prev over 1e-2 .. 1e2, plus_velocity mixed, v_boundary absent and present -- for dense random
stand-ins (with a P row that is all zero, a P row with zeros inside its range and a D_1_0 column that is all zero) and
for the reference's operators (oracle/fiber_fd.py: P block diagonal, D_1_0 banded).  It is sharp: every planted defect
misses its bound by at least DEFECT_FACTOR x K on some entry.  And the restatement is the operation the project's float64
oracle states (oracle.fiber_container_matvec, apply_fiber_force, fiber_apply_preconditioner): they agree to 1e-12."""
import numpy as np
import pytest

import fiber_gemv_reference as fg
import oracle as orc
from oracle import fiber_fd

NODES = (4, 5, 7, 8, 14, 15, 16, 17, 31, 32, 33, 48, 64, 96, 128)
# the smallest factor by which a defect must miss its bound (ratio / K); every defect below misses by far more
DEFECT_FACTOR = 1e6


def alternating(nodes, reps):
    """small and large node counts alternating: 4, 128, 5, 96, ... repeated reps times"""
    s = sorted(nodes)
    out = []
    for i in range((len(s) + 1) // 2):
        out += [s[i]] + ([s[-1 - i]] if len(s) - 1 - i > i else [])
    return out * reps


def straight_fibers(rng, n_nodes):
    lengths = rng.uniform(0.5, 2.0, len(n_nodes))
    pos = []
    for n, L in zip(n_nodes, lengths):
        t = rng.normal(size=3)
        pos.append(rng.uniform(-3, 3, 3) + np.linspace(0, L, n)[:, None] * t / np.linalg.norm(t))
    return dict(pos=np.concatenate(pos), n_nodes=[int(n) for n in n_nodes], lengths=list(lengths))


def inputs(rng, n_nodes):
    """x (4 N_f,) and v (N_f, 3), each fiber's scaled by its own 10^U(-3, 3); v_boundary (n_fibers, 7)"""
    sx, sv = (10.0 ** rng.uniform(-3, 3, len(n_nodes)) for _ in range(2))
    x = np.concatenate([rng.normal(size=4 * n) * s for n, s in zip(n_nodes, sx)])
    v = rng.normal(size=(int(np.sum(n_nodes)), 3)) * np.repeat(sv, n_nodes)[:, None]
    vb = rng.normal(size=(len(n_nodes), 7)) * 10.0 ** rng.uniform(-3, 3, (len(n_nodes), 1))
    return x, v, vb


def _per_fiber(rng, n_nodes, ops):
    xs = rng.normal(size=(int(np.sum(n_nodes)), 3))
    ops["xs"] = xs / np.linalg.norm(xs, axis=1)[:, None]
    ops["length_prev"] = list(10.0 ** rng.uniform(-2, 2, len(n_nodes)))
    ops["plus"] = [int(p) for p in rng.integers(0, 2, len(n_nodes))]
    return ops


def dense_case(seed, nodes=NODES, reps=2):
    """family (a): dense random stand-ins of the reference's shapes, plus one P with an all-zero row (n = 17), one P
    whose row 40 has zeros at both ends and inside its range (n = 33) and one D_1_0 with an all-zero column (n = 15).
    A_^-1 is a dense random stand-in too: the kernel is plain linear algebra.  Returns (fib, ops, A_inv, x, v, vb)."""
    rng = np.random.default_rng(seed)
    n_nodes = alternating(nodes, reps)
    fib = straight_fibers(rng, n_nodes)
    ops = dict(n_nodes=n_nodes, A=[], force=[], D_1_0={}, P={})
    A_inv = []
    for n in n_nodes:
        ops["A"].append(rng.normal(size=(4 * n, 4 * n)))
        ops["force"].append(rng.normal(size=(3 * n, 4 * n)))
        A_inv.append(rng.normal(size=(4 * n, 4 * n)))
        if n not in ops["D_1_0"]:
            ops["D_1_0"][n] = rng.normal(size=(n, n))
            ops["P"][n] = rng.normal(size=(4 * n - 14, 4 * n))
    if 17 in ops["P"]:
        ops["P"][17][5] = 0.0
    if 33 in ops["P"]:
        ops["P"][33][40, :7] = 0.0
        ops["P"][33][40, -3:] = 0.0
        ops["P"][33][40, 20:50:3] = 0.0
    if 15 in ops["D_1_0"]:
        ops["D_1_0"][15][:, 3] = 0.0
    _per_fiber(rng, n_nodes, ops)
    return (fib, ops, A_inv) + inputs(rng, n_nodes)


def reference_case(seed, clamp, pin, nodes=tuple(n for n in NODES if n >= 8), reps=2):
    """family (b): the reference's operators (oracle/fiber_fd.py) on straight fibers, with clamp / pin fractions;
    length_prev and plus_velocity then redrawn over the ranges above (the GEMVs take them as inputs).  A_^-1 is numpy's
    inverse of A_.  Returns (fib, ops, A_inv, x, v, vb)."""
    rng = np.random.default_rng(seed)
    n_nodes = alternating(nodes, reps)
    fib = straight_fibers(rng, n_nodes)
    ops = fiber_fd.suspension_operators(fib["pos"], n_nodes, fib["lengths"], eta=0.9, seed=seed, clamp_fraction=clamp,
                                        pin_fraction=pin)
    xs = ops["xs"]
    _per_fiber(rng, n_nodes, ops)
    ops["xs"] = xs
    return (fib, ops, [np.linalg.inv(A) for A in ops["A"]]) + inputs(rng, n_nodes)


CASES = {"dense": lambda: dense_case(1), "reference_0": lambda: reference_case(2, 0.0, 0.0),
         "reference_half": lambda: reference_case(3, 0.5, 0.5)}


@pytest.fixture(scope="module", params=sorted(CASES))
def case(request):
    return request.param, CASES[request.param]()


def _worst(r, K):
    return float(np.max(r / K))


def test_nonzero_ranges_follow_the_host_planning():
    M = np.array([[0.0, 1.0, 0.0, 2.0, 0.0], [0.0] * 5, [3.0, 0.0, 0.0, 0.0, 0.0]])
    assert fg.nonzero_ranges(M, 1)[0].tolist() == [1, 0, 0] and fg.nonzero_ranges(M, 1)[1].tolist() == [4, 0, 1]
    assert fg.nonzero_ranges(M, 0)[0].tolist() == [2, 0, 0, 0, 0]
    assert fg.nonzero_ranges(M, 0)[1].tolist() == [3, 1, 0, 1, 0]


def test_slices_follow_the_kernels_order():
    # a sum whose value depends on the order: slice q holds columns q, q + 8, ...; then slices 0 .. 7 in turn
    t = np.zeros((1, 24))
    t[0, 0], t[0, 8], t[0, 1] = 1.0, 2.0 ** -53, -1.0
    p = fg.slice_partials(t)
    assert p[0, 0] == 1.0 + 2.0 ** -53 and p[1, 0] == -1.0 and fg.slice_sum(p)[0] == 0.0
    # drop_tail_column: 20 columns -> slices 0 .. 3 have 3 columns (a tail of 3), 4 .. 7 two
    t = np.ones((1, 20))
    assert fg.slice_partials(t, "drop_tail_column")[:, 0].tolist() == [2, 2, 2, 2, 1, 1, 1, 1]
    # 64 columns: every slice has 8 columns, no tail
    assert fg.slice_partials(np.ones((1, 64)), "drop_tail_column")[:, 0].tolist() == [8] * 8


def test_float64_meets_its_bounds(case):
    assert np.finfo(np.longdouble).nmant >= 63
    name, (fib, ops, A_inv, x, v, vb) = case
    worst = {}
    for mode, fn, args in ((1, fg.fiber_force, (ops["force"], x, ops["n_nodes"])),
                           (0, fg.fiber_precondition, (A_inv, x, ops["n_nodes"])),
                           (2, fg.fiber_matvec, (ops, x, v, None)),
                           (2, fg.fiber_matvec, (ops, x, v, vb))):
        K = fg.k_rows(ops, mode)
        r = fg.ratio(fn(*args, dtype=np.float64), *fg.ext_and_scale(fn, *args))
        assert np.isfinite(r).all() and (r <= K).all(), (name, mode, np.unravel_index(r.argmax(), r.shape), r.max())
        worst[mode] = max(worst.get(mode, 0.0), _worst(r, K))
    print(f"\n{name}: float64 worst ratio / K: " + ", ".join(f"MODE {m} {w:.3f}" for m, w in sorted(worst.items())))


def test_planted_structure_is_there():
    _, ops, _, _, _, _ = dense_case(1)
    lo, hi = fg.nonzero_ranges(ops["P"][17], 1)
    assert lo[5] == 0 and hi[5] == 0
    lo, hi = fg.nonzero_ranges(ops["P"][33], 1)
    assert lo[40] == 7 and hi[40] == 4 * 33 - 3
    lo, hi = fg.nonzero_ranges(ops["D_1_0"][15], 0)
    assert lo[3] == 0 and hi[3] == 0
    # the reference's P is block diagonal and its D_1_0 banded: the walked ranges really narrow
    _, rops, _, _, _, _ = reference_case(2, 0.0, 0.0)
    for n in rops["P"]:
        lo, hi = fg.nonzero_ranges(rops["P"][n], 1)
        assert (hi - lo).max() == n
        dlo, dhi = fg.nonzero_ranges(rops["D_1_0"][n], 0)
        assert (dhi - dlo).max() < n or n <= 8


def _defect_case(defect, name, fib, ops, A_inv, x, v, vb):
    """(f64 with the defect, ext, S, K) on the mode the defect lives in"""
    if defect == "force_scatter_transposed":
        fn, args, mode = fg.fiber_force, (ops["force"], x, ops["n_nodes"]), 1
    else:
        fn, args, mode = fg.fiber_matvec, (ops, x, v, vb), 2
    return fn(*args, dtype=np.float64, defect=defect), *fg.ext_and_scale(fn, *args), fg.k_rows(ops, mode)


@pytest.mark.parametrize("defect", fg.DEFECTS)
def test_criterion_catches_planted_defects(case, defect):
    name, c = case
    bad, e, S, K = _defect_case(defect, name, *c)
    f = _worst(fg.ratio(bad, e, S), K)
    print(f"\n{name}, {defect}: misses its bound by {f:.3g} x K")
    assert f > DEFECT_FACTOR, (name, defect, f)


@pytest.mark.parametrize("defect", fg.GEMV_DEFECTS)
def test_gemv_defects_are_caught_in_every_mode(defect):
    _, ops, A_inv, x, v, vb = dense_case(1)
    for mode, fn, args in ((1, fg.fiber_force, (ops["force"], x, ops["n_nodes"])),
                           (0, fg.fiber_precondition, (A_inv, x, ops["n_nodes"]))):
        f = _worst(fg.ratio(fn(*args, dtype=np.float64, defect=defect), *fg.ext_and_scale(fn, *args)),
                   fg.k_rows(ops, mode))
        assert f > DEFECT_FACTOR, (defect, mode, f)


def test_ext_agrees_with_the_float64_oracle(case):
    name, (fib, ops, A_inv, x, v, vb) = case
    rel = lambda a, b: float(np.abs(np.asarray(a, dtype=np.float64) - b).max() / np.abs(b).max())
    for w in (None, vb):
        assert rel(fg.fiber_matvec(ops, x, v, w), orc.fiber_container_matvec(ops, x, v, w)) <= 1e-12, (name, w)
    assert rel(fg.fiber_force(ops["force"], x, ops["n_nodes"]), orc.apply_fiber_force(ops["force"], x,
                                                                                       ops["n_nodes"])) <= 1e-12
    # the oracle's preconditioner is an LU solve: tie MODE 0 to it on well-conditioned matrices
    rng = np.random.default_rng(9)
    A = [np.eye(4 * n) + 0.3 * rng.normal(size=(4 * n, 4 * n)) / np.sqrt(4 * n) for n in ops["n_nodes"]]
    y = fg.fiber_precondition([np.linalg.inv(a) for a in A], x, ops["n_nodes"])
    assert rel(y, orc.fiber_apply_preconditioner(A, x, ops["n_nodes"])) <= 1e-12

"""Tests of skb_flow_build_fiber_operators (include/skelly_b200_flow.h): the per-fiber operators A_, force_operator_,
xs_ and A_^-1 built on the device from positions, lengths and per-fiber scalars.

The operators are held to the oracle's statement-by-statement restatement of update_derivatives /
update_linear_operator / apply_bc_rectangular / update_force_operator (oracle/fiber_fd.py::FiberOperators) evaluated
in np.longdouble on the same float64 inputs, and the inverse to a long-double Gauss-Jordan inverse of the device's
own A_.  The criteria are anchored to what a correct FP64 computation achieves, so that they tell a correct kernel
from a slightly wrong one:

* operators (A_, force_operator_, xs_): |dev - ext| <= C_OPS u S entry by entry, u = 2^-53, S the same computation
  on absolute values (FiberOperators(absolute=True)); a structural zero (S = 0) must be exactly zero.  A whole-matrix
  rel_max would hold a boundary row of A_ (row magnitudes span 2e2 .. 4e8 at n = 128) to ~1e-6 of its own size.
* inverse: for each of the 16 n x n blocks of A_^-1, the relative Frobenius error against the extended inverse is
  <= K_INV x that of numpy's LAPACK inverse (np.linalg.inv, standing in for Eigen's PartialPivLU::inverse) of the same
  matrix, + FLOOR_INV (K_INV_RANGES for the parameter-range builds, see below).  A 1e-16 cond(A) bound admits 1e-5
  at cond 1e11; a correct FP64 inverse errs by ~1e-10 there.
* the inverse's consumer (apply_fiber_preconditioner, fiber_gemv_kernel<0>): y = A_^-1 x is held to the device's own
  A_^-1, |y - A_^-1 x| <= C_OPS u |A_^-1| |x| entry by entry, A_^-1 x in long double.  Holding y instead to the
  extended inverse at K_INV x the error of LAPACK's inverse applied in FP64 fails the correct host restatement: its
  error on A^-1 x reached 21x LAPACK's for one matrix (dt = 1e-5, n = 64) over 8 random right-hand sides, 34x on one,
  although its blockwise inverse error there is within the bound.  The blockwise check is what holds the inverse.

The CPU tests below show every criterion attainable and sharp on every matrix the GPU tests use: the float64 oracle,
LAPACK and a host restatement of the kernel's Gauss-Jordan (fiber_fd.gauss_jordan_inverse) pass; planted defects
fail.  Calibration (x86 host, np.longdouble = 64-bit mantissa; "curved" is the 16-fiber build at dt = 5e-3, the
parameter ranges are two 16-fiber builds at dt = 1e-5 and 1e-1; device figures on an H100 SXM 80 GB at a 400 W power
limit):

* operators: the float64 oracle reaches 4.6 u S, the device 5.5 u S; C_OPS = 8.  One boundary row of A_ scaled by
  (1 + delta) is caught from delta = 1e-14 (1e-15 on some fibers) on every fiber, against ~1e-6 for rel_max at
  n = 128.  Dropping the (c0 + c1) xss diagonal term of one block fails on every curved fiber.  The extended
  inverse's own error (the correction of a second refinement step) is below 1 % of LAPACK's blockwise error.
* inverse, curved build: the host restatement, also with its pivot reciprocals one rounding off, is within 8.6x of
  LAPACK blockwise (the device: 7.3x, at n = 64), so K_INV = 16.  Planted defects, as multiples of LAPACK's error: a
  pivot reciprocal off by 1e-13 (>= 26.6x) and no pivoting (>= 1 600x) fail on every matrix; a 32-row pivot window
  fails on every matrix with n >= 24 and changes nothing at n = 8 (at n = 16: 9.1x).
* inverse, parameter ranges: Gauss-Jordan is not LAPACK's LU-based inverse, and on the stiff matrices of dt = 1e-5
  its blockwise error scatters: the restatement reaches 21.9x LAPACK's (n = 96), and 32.8x (n = 16) with one pivot
  reciprocal a rounding off.  A bound at K_INV there would fail a correct kernel, so these builds are held at
  K_INV_RANGES = 128 (the device: 15.8x at worst, n = 24).  No pivoting (>= 909x) and a 32-row window at n >= 24
  (>= 199x) still fail on every matrix; the 1e-13 reciprocal defect (6.9x .. 4 550x) passes on 13 of 32 matrices, so
  the curved build is what holds the reciprocal.

Host time: the extended references cost ~3 s per n = 128 fiber (Gauss-Jordan and two refinement steps in long
double); the CPU tests of this file take ~70 s, the GPU tests ~85 s of host time.  Where np.longdouble is IEEE quad in
software (aarch64) every long-double operation is emulated; that has not been measured and is expected to cost an
order of magnitude more.  The extended reference refuses to run where np.longdouble is plain double.
"""
import os
import shutil
import subprocess

import numpy as np
import pytest
import scipy.linalg

import oracle as orc
import skellysim_b200 as skb
from oracle import fiber_fd
from conftest import rel_l2, rel_max
from test_gpu_flow import ft_of, load

NODES = (8, 16, 24, 32, 48, 64, 96, 128)
ETA, DT = 0.9, 5e-3
RANGE_DTS = (1e-5, 1e-1)                   # time steps of the parameter-range builds
U = 2.0 ** -53
C_OPS = 8.0                                 # operators: |dev - ext| <= C_OPS u S
K_INV = 16.0                                # inverse: blockwise error <= K x LAPACK's + FLOOR_INV, K = K_INV for
K_INV_RANGES = 128.0                        # the curved build, K_INV_RANGES for the parameter-range builds
FLOOR_INV = 4 * U
CLUSTER = {8: 1, 16: 1, 24: 1, 32: 1, 48: 2, 64: 3, 96: 6, 128: 10}  # fiber_build.cuh: inverse_cluster_size(4n)


def curved_fibers(seed, n_nodes):
    """Smooth curved fibers (an arc of a random helix per fiber), their lengths and random per-fiber scalars."""
    rng = np.random.default_rng(seed)
    pos, lengths = [], []
    for n in n_nodes:
        L = rng.uniform(0.6, 1.6)
        s = np.linspace(0.0, L, n)
        k, tau = rng.uniform(0.3, 1.5), rng.uniform(-1.0, 1.0)
        a = np.hypot(k, tau)                       # arc-length parametrised helix of curvature k, torsion tau
        c = np.stack([k / a ** 2 * np.cos(a * s), k / a ** 2 * np.sin(a * s), tau / a * s], axis=1)
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        pos.append(rng.uniform(-4, 4, 3) + c @ q.T)
        lengths.append(L)
    nf = len(n_nodes)
    combos = np.arange(nf) % 4                      # every (minus clamped, plus hinged) combination
    prm = dict(length_prev=np.array(lengths) * rng.uniform(0.95, 1.05, nf), bending_rigidity=rng.uniform(1e-3, 1e-2, nf),
               radius=rng.uniform(5e-3, 2e-2, nf), penalty_param=rng.uniform(100.0, 800.0, nf),
               beta_tstep=rng.uniform(0.5, 1.5, nf), minus_clamped=(combos & 1).astype(np.int32),
               plus_hinged=(combos >> 1).astype(np.int32))
    fib = dict(pos=np.concatenate(pos), n_nodes=[int(n) for n in n_nodes], lengths=lengths,
               forces=rng.uniform(-1, 1, (int(np.sum(n_nodes)), 3)))
    return fib, prm


def range_fibers(seed, build):
    """Two fibers per node count for one of two builds (build = 0, 1): over both builds every node count meets all four
    boundary-condition combinations.  Lengths 0.05 .. 20 and bending rigidities 1e-4 .. 1e-1 on log-spaced grids,
    length_prev 5 .. 25 % off the length, straight fibers and strongly curved ones (a helix turning 1 .. 4 rad).  A
    straight fiber clamped at the minus end and hinged at the plus end is singular: that combination is always curved."""
    rng = np.random.default_rng(seed)
    nf = 2 * len(NODES)
    lengths, E = np.geomspace(0.05, 20.0, nf), np.geomspace(1e-4, 1e-1, nf)
    rng.shuffle(lengths)
    rng.shuffle(E)
    pos, n_nodes, combos = [], [], []
    for i, n in enumerate(NODES):
        for j in range(2):
            f, combo = len(n_nodes), (2 * build + j + i) % 4
            L = lengths[f]
            s = np.linspace(0.0, L, n)
            if combo != 3 and (i + j) % 2 == 0:
                c = s[:, None] * np.array([0.0, 0.0, 1.0])
            else:
                k = rng.uniform(1.0, 4.0) / L
                tau = rng.uniform(-1.0, 1.0) * k
                a = np.hypot(k, tau)
                c = np.stack([k / a ** 2 * np.cos(a * s), k / a ** 2 * np.sin(a * s), tau / a * s], axis=1)
            q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
            pos.append(rng.uniform(-4, 4, 3) + c @ q.T)
            n_nodes.append(n)
            combos.append(combo)
    combos = np.array(combos)
    prm = dict(length_prev=lengths * rng.choice([-1, 1], nf) * rng.uniform(0.05, 0.25, nf) + lengths,
               bending_rigidity=E, radius=rng.uniform(5e-3, 2e-2, nf), penalty_param=rng.uniform(100.0, 800.0, nf),
               beta_tstep=rng.uniform(0.5, 1.5, nf), minus_clamped=(combos & 1).astype(np.int32),
               plus_hinged=(combos >> 1).astype(np.int32))
    fib = dict(pos=np.concatenate(pos), n_nodes=n_nodes, lengths=list(lengths), forces=rng.uniform(-1, 1, (sum(n_nodes), 3)))
    return fib, prm


def fiber_operators(fib, prm, dt=DT, f0=0, f1=None, **kw):
    """oracle FiberOperators of fibers [f0, f1); kw: dtype / absolute"""
    f1 = len(fib["n_nodes"]) if f1 is None else f1
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
    return [fiber_fd.FiberOperators(fib["pos"][off[f]:off[f + 1]], fib["lengths"][f],
                                    bending_rigidity=prm["bending_rigidity"][f], radius=prm["radius"][f], eta=ETA,
                                    dt=dt, length_prev=prm["length_prev"][f], minus_clamped=bool(prm["minus_clamped"][f]),
                                    plus_pinned=bool(prm["plus_hinged"][f]), penalty_param=prm["penalty_param"][f],
                                    beta_tstep=prm["beta_tstep"][f], **kw) for f in range(f0, f1)]


def oracle_ops(fib, prm, f0=0, f1=None, dt=DT):
    fos = fiber_operators(fib, prm, dt, f0, f1)
    ops = dict(n_nodes=[fo.n for fo in fos], A=[fo.A for fo in fos], force=[fo.force_operator for fo in fos],
               xs=np.concatenate([fo.xs for fo in fos]) if fos else np.zeros((0, 3)),
               length_prev=[fo.length_prev for fo in fos], plus=[fo.plus_bc_velocity for fo in fos], D_1_0={}, P={})
    for fo in fos:
        ops["D_1_0"][fo.n], ops["P"][fo.n] = fo.mats["D_1_0"], fo.mats["P_downsample_bc"]
    return ops


def set_classes(fl, n_nodes):
    for n in sorted(set(n_nodes)):
        m = fiber_fd.compute_matrices(n)
        fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])


def build(fl, prm, sl=slice(None), dt=DT):
    fl.build_fiber_operators(*(prm[k][sl] for k in ("length_prev", "bending_rigidity", "radius", "penalty_param",
                                                    "beta_tstep", "minus_clamped", "plus_hinged")), dt, ETA)


def empty_shell_body(seed=0, n_shell=0, n_body=0):
    from test_gpu_flow import make_system
    _, shell, body = make_system(seed, 0, n_shell, n_body, 1 if n_body else 0)
    return shell, body


# ---- the criteria ----------------------------------------------------------------------------------------------------

def op_ratio(got, ext, S):
    """max over the entries of |got - ext| / (u S); a structural zero (S = 0) counts 0 if exactly zero, inf if not."""
    d = np.abs(np.asarray(got, dtype=np.float64).astype(np.longdouble) - ext).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(S > 0, d / (U * S), np.where(d == 0, 0.0, np.inf))
    return float(np.max(r))          # (NaN in `got` gives NaN, which fails every <= test)


def block_errors(X, X_ext):
    """relative Frobenius error of each of the 16 n x n blocks of X against X_ext"""
    n = X.shape[0] // 4
    D = (np.asarray(X).astype(np.longdouble) - X_ext).astype(np.float64)
    Xe = X_ext.astype(np.float64)
    return np.array([np.linalg.norm(D[a * n:(a + 1) * n, b * n:(b + 1) * n]) /
                     np.linalg.norm(Xe[a * n:(a + 1) * n, b * n:(b + 1) * n]) for a in range(4) for b in range(4)])


def inverse_k(case):
    return K_INV if case == "curved" else K_INV_RANGES


def inverse_ok(X, X_ext, X_lapack, K):
    return bool(np.all(block_errors(X, X_ext) <= K * block_errors(X_lapack, X_ext) + FLOOR_INV))


def inverse_ratio(X, X_ext, X_lapack):
    """worst blockwise error of X as a multiple of LAPACK's (reported beside the criterion)"""
    return float(np.max(block_errors(X, X_ext) / block_errors(X_lapack, X_ext)))


def gemv_ratio(y, X, x):
    """max over the entries of |y - X x| / (u |X| |x|), X x evaluated in long double: how far y is from the matrix X
    it was computed from, in units of the error scale of any FP64 evaluation order"""
    xe = np.asarray(x, dtype=np.float64).astype(np.longdouble)
    return op_ratio(y, np.asarray(X, dtype=np.float64).astype(np.longdouble) @ xe, np.abs(X) @ np.abs(x))


def check_operators(got, ext, S, label):
    """A_, force_operator_ and xs_ of every fiber within C_OPS u S; returns the worst ratio"""
    worst = 0.0
    off = np.concatenate([[0], np.cumsum([a.shape[0] // 4 for a in got["A"]])])
    for f in range(len(got["A"])):
        for k, g in (("A", got["A"][f]), ("force", got["force"][f]), ("xs", got["xs"][off[f]:off[f + 1]])):
            r = op_ratio(g, ext[k][f], S[k][f])
            assert r <= C_OPS, (label, f, k, r)
            worst = max(worst, r)
    return worst


# ---- the cases -------------------------------------------------------------------------------------------------------

def extended_ops(fib, prm, dt):
    """the long-double operators (ext) and their error scales (S) of every fiber, keyed like get_fiber_operators"""
    ext = fiber_operators(fib, prm, dt, dtype=np.longdouble)
    S = fiber_operators(fib, prm, dt, absolute=True)
    return ({"A": [e.A for e in ext], "force": [e.force_operator for e in ext], "xs": [e.xs for e in ext]},
            {"A": [s.A for s in S], "force": [s.force_operator for s in S], "xs": [s.xs for s in S]})


@pytest.fixture(scope="module")
def system():
    n_nodes = list(NODES) * 2
    np.random.default_rng(7).shuffle(n_nodes)
    fib, prm = curved_fibers(11, n_nodes)
    return fib, prm, oracle_ops(fib, prm)


@pytest.fixture(scope="module")
def cases(system):
    """every build the GPU tests hold to the extended reference: (fib, prm, dt, ext, S, float64 oracle operators)"""
    out = {}
    for name, (fib, prm), dt in [("curved", system[:2], DT)] + [
            (f"ranges{b}", range_fibers(21 + b, b), RANGE_DTS[b]) for b in range(len(RANGE_DTS))]:
        ext, S = extended_ops(fib, prm, dt)
        out[name] = dict(fib=fib, prm=prm, dt=dt, ext=ext, S=S, fp64=fiber_operators(fib, prm, dt))
    return out


@pytest.fixture(scope="module")
def oracle_inverses(cases):
    """per case and fiber: the extended inverse of the float64 oracle's A_, its refinement correction and LAPACK's"""
    out = {}
    for name, c in cases.items():
        out[name] = []
        for fo in c["fp64"]:
            X, dX = fiber_fd.extended_inverse(fo.A)
            out[name].append(dict(X=X, dX=dX, lapack=np.linalg.inv(fo.A)))
    return out


# ---- CPU: the criteria are attainable and sharp ----------------------------------------------------------------------

def test_extended_inverse_is_accurate(cases, oracle_inverses):
    # long double must be wider than double, and the extended inverse must be exact to 1 % of the FP64 errors measured
    assert np.finfo(np.longdouble).nmant >= 63
    for name, invs in oracle_inverses.items():
        for f, inv in enumerate(invs):
            corr = block_errors(inv["X"] + inv["dX"], inv["X"])
            lap = block_errors(inv["lapack"], inv["X"])
            assert np.all(corr <= 0.01 * lap), (name, f, (corr / lap).max())


def test_operator_criterion_holds_for_the_fp64_oracle(cases):
    worst = {}
    for name, c in cases.items():
        got = dict(A=[fo.A for fo in c["fp64"]], force=[fo.force_operator for fo in c["fp64"]],
                   xs=np.concatenate([fo.xs for fo in c["fp64"]]))
        worst[name] = check_operators(got, c["ext"], c["S"], name)
    print("fp64 oracle |dA|/(u S), worst:", worst)


def test_inverse_criterion_holds_for_lapack_and_the_restatement(cases, oracle_inverses):
    # the restatement, and the restatement with its pivot reciprocals one rounding off (the spread of a correct FP64
    # Gauss-Jordan under a different rounding, such as the kernel's fused multiply-adds)
    worst = {}
    for name, c in cases.items():
        K = inverse_k(name)
        for f, (fo, inv) in enumerate(zip(c["fp64"], oracle_inverses[name])):
            assert inverse_ok(inv["lapack"], inv["X"], inv["lapack"], K)
            for rel in (0.0, U, -U):
                G = fiber_fd.gauss_jordan_inverse(fo.A, recip_rel_err=rel)
                r = inverse_ratio(G, inv["X"], inv["lapack"])
                assert inverse_ok(G, inv["X"], inv["lapack"], K), (name, f, fo.n, rel, r)
                worst[(name, fo.n)] = max(worst.get((name, fo.n), 0.0), r)
            x = np.random.default_rng(f).normal(size=4 * fo.n)
            assert gemv_ratio(G @ x, G, x) <= C_OPS
    print("\nhost Gauss-Jordan / LAPACK blockwise, worst per n:", {k: round(v, 1) for k, v in worst.items()})


DEFECTS = {"recip 1e-13": dict(recip_rel_err=1e-13), "pivot window 32": dict(pivot_window=32),
           "no pivoting": dict(pivoting=False)}


def test_inverse_criterion_catches_planted_defects(cases, oracle_inverses):
    # every defect fails on every matrix, except: a 32-row pivot window changes nothing at n = 8 and little at n = 16,
    # and a pivot reciprocal off by 1e-13 hides in the looser bound of the parameter-range builds (reported, not held)
    ratios = {}
    for name, c in cases.items():
        for f, (fo, inv) in enumerate(zip(c["fp64"], oracle_inverses[name])):
            for d, kw in DEFECTS.items():
                G = fiber_fd.gauss_jordan_inverse(fo.A, **kw)
                ok = inverse_ok(G, inv["X"], inv["lapack"], inverse_k(name))
                r = inverse_ratio(G, inv["X"], inv["lapack"])
                ratios.setdefault((name, d), []).append((fo.n, round(r, 1), ok))
                must_fail = (d != "pivot window 32" or fo.n >= 24) and (name == "curved" or d != "recip 1e-13")
                assert not (must_fail and ok), (name, d, fo.n, r)
    print("\ndefect / LAPACK blockwise, smallest:", {k: min(r for _, r, _ in v) for k, v in ratios.items()},
          "; passing:", {k: [(n, r) for n, r, ok in v if ok] for k, v in ratios.items()})


def test_operator_criterion_catches_planted_defects(cases):
    worst_delta = {}
    for name, c in cases.items():
        for f, fo in enumerate(c["fp64"]):
            n, A_ext, S = fo.n, c["ext"]["A"][f], c["S"]["A"][f]
            # one boundary row scaled by (1 + delta): the smallest power of ten caught, over the 14 rows
            for t in range(14):
                row = 4 * n - 14 + t
                for e in range(3, 17):
                    if op_ratio(fo.A[row] * (1 + 10.0 ** -e), A_ext[row], S[row]) <= C_OPS:
                        break
                assert e > 3, (name, f, t)
                worst_delta[(name, n)] = max(worst_delta.get((name, n), 0.0), 10.0 ** -(e - 1))
            # the (c0 + c1) xss diagonal term of block (a, 3) dropped, a = f % 3
            a = int(np.argmax(np.abs(fo.xss).max(axis=0)))
            if np.abs(fo.xss).max() * fo.length > 0.5:          # a curved fiber
                A = fo.A.copy()
                A[:4 * n - 14, 3 * n:] += fo.mats["P_downsample_bc"][:, a * n:(a + 1) * n] @ np.diag((fo.c_0 + fo.c_1) * fo.xss[:, a])
                assert op_ratio(A, A_ext, S) > C_OPS, (name, f, n)
    print("smallest boundary-row delta caught, worst over rows:", worst_delta)
    assert max(worst_delta.values()) <= 1e-8


def test_pivoting_is_exercised_for_every_cluster_size(cases):
    # partial pivoting must reach >= 32 rows below the diagonal and take pivots from the 14 boundary rows in the matrices
    # of every cluster size of fiber_inverse_kernel
    far, boundary = set(), set()
    for c in cases.values():
        for fo in c["fp64"]:
            m = 4 * fo.n
            _, piv = scipy.linalg.lu_factor(fo.A, check_finite=False)
            rows = np.arange(m)
            for k, p in enumerate(piv):
                rows[[k, p]] = rows[[p, k]]
                if p - k >= 32:
                    far.add(CLUSTER[fo.n])
                if rows[k] >= m - 14:
                    boundary.add(CLUSTER[fo.n])
    assert far == boundary == set(CLUSTER.values()), (far, boundary)


# ---- GPU -------------------------------------------------------------------------------------------------------------

def check_inverse(got, x, y, label, K):
    """A_^-1 of every fiber blockwise against the extended inverse of the device's own A_, and y = A_^-1 x of
    apply_fiber_preconditioner against the device's A_^-1; returns the worst device / LAPACK blockwise ratio per n"""
    worst, off = {}, 0
    for f, (A, X) in enumerate(zip(got["A"], got["A_inv"])):
        m = A.shape[0]
        X_ext, dX = fiber_fd.extended_inverse(A)
        lap = np.linalg.inv(A)
        e_lap = block_errors(lap, X_ext)
        assert np.all(block_errors(X_ext + dX, X_ext) <= 0.01 * e_lap), (label, f, "extended inverse")
        assert inverse_ok(X, X_ext, lap, K), (label, f, m // 4, inverse_ratio(X, X_ext, lap))
        worst[m // 4] = max(worst.get(m // 4, 0.0), inverse_ratio(X, X_ext, lap))
        r = gemv_ratio(y[off:off + m], X, x[off:off + m])
        assert r <= C_OPS, (label, f, m // 4, "preconditioner", r)
        off += m
    return worst


def build_and_read(fib, prm, dt, x):
    shell, body = empty_shell_body()
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])
        build(fl, prm, dt=dt)
        got = fl.get_fiber_operators()
        y = fl.apply_fiber_preconditioner(x) if x is not None else None
    return got, y


@pytest.mark.gpu
def test_build_matches_oracle_operators_and_inverse(system, cases):
    fib, prm, ops = system
    x = np.random.default_rng(8).normal(size=4 * fib["pos"].shape[0])
    got, y = build_and_read(fib, prm, DT, x)
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
    assert rel_max(got["xs"], ops["xs"]) <= 1e-12
    for f, n in enumerate(fib["n_nodes"]):
        A_ref = ops["A"][f]
        assert rel_max(got["A"][f], A_ref) <= 1e-12, (f, n, rel_max(got["A"][f], A_ref))
        assert rel_max(got["force"][f], ops["force"][f]) <= 1e-12, (f, n)
        assert rel_max(got["xs"][off[f]:off[f + 1]], ops["xs"][off[f]:off[f + 1]]) <= 1e-12, (f, n)
        X, A = got["A_inv"][f], got["A"][f]
        res = np.linalg.norm(A @ X - np.eye(4 * n)) / (np.linalg.norm(A) * np.linalg.norm(X))
        assert res <= 1e-12, (f, n, res)
    c = cases["curved"]
    print("\ncurved: device |dA|/(u S) worst", check_operators(got, c["ext"], c["S"], "curved"),
          "; device / LAPACK blockwise, worst per n", check_inverse(got, x, y, "curved", K_INV))


@pytest.mark.gpu
@pytest.mark.parametrize("b", range(len(RANGE_DTS)))
def test_build_over_parameter_ranges(cases, b):
    c = cases[f"ranges{b}"]
    x = np.random.default_rng(9 + b).normal(size=4 * c["fib"]["pos"].shape[0])
    got, y = build_and_read(c["fib"], c["prm"], c["dt"], x)
    print(f"\nranges{b} (dt = {c['dt']}): device |dA|/(u S) worst",
          check_operators(got, c["ext"], c["S"], f"ranges{b}"),
          "; device / LAPACK blockwise, worst per n", check_inverse(got, x, y, f"ranges{b}", K_INV_RANGES))


def singular_set(with_singular):
    """range_fibers(31, 0) and, after the two fibers of every node count, a straight fiber clamped at the minus end and
    hinged at the plus end (its A_ is singular up to rounding: cond ~1e18)"""
    fib, prm = range_fibers(31, 0)
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
    keys = list(prm)
    pos, n_nodes, lengths, p, ordinary = [], [], [], {k: [] for k in keys}, []
    for f, n in enumerate(fib["n_nodes"]):
        ordinary.append(len(n_nodes))
        pos.append(fib["pos"][off[f]:off[f + 1]])
        n_nodes.append(n)
        lengths.append(fib["lengths"][f])
        for k in keys:
            p[k].append(prm[k][f])
        if with_singular and f % 2 == 1:
            pos.append(np.array([0.5, -1.0, 2.0]) + np.linspace(0.0, 1.0, n)[:, None] * np.array([0.6, 0.0, 0.8]))
            n_nodes.append(n)
            lengths.append(1.0)
            for k, v in dict(length_prev=1.0, bending_rigidity=1e-2, radius=1e-2, penalty_param=500.0, beta_tstep=1.0,
                             minus_clamped=1, plus_hinged=1).items():
                p[k].append(v)
    p = {k: np.array(v, dtype=prm[k].dtype) for k, v in p.items()}
    fib = dict(pos=np.concatenate(pos), n_nodes=n_nodes, lengths=lengths)
    return fib, p, ordinary


@pytest.mark.gpu
def test_singular_fiber_leaves_the_others_untouched():
    fib, prm, ordinary = singular_set(True)
    fib0, prm0, _ = singular_set(False)
    singular = sorted(set(range(len(fib["n_nodes"]))) - set(ordinary))
    for f in singular:
        assert np.linalg.cond(fiber_operators(fib, prm, DT, f, f + 1)[0].A) > 1e15
    got, _ = build_and_read(fib, prm, DT, None)       # the call succeeds
    ref, _ = build_and_read(fib0, prm0, DT, None)
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
    off0 = np.concatenate([[0], np.cumsum(fib0["n_nodes"])])
    for f0, f in enumerate(ordinary):
        for k in ("A", "force", "A_inv"):
            assert np.array_equal(got[k][f], ref[k][f0]), (f, k)
        assert np.array_equal(got["xs"][off[f]:off[f + 1]], ref["xs"][off0[f0]:off0[f0 + 1]]), f


@pytest.mark.gpu
def test_apply_matvec_after_build(system):
    fib, prm, ops = system
    shell, body = empty_shell_body(3, 400, 120)
    rng = np.random.default_rng(5)
    nf, ns = fib["pos"].shape[0], shell["pos"].shape[0]
    x = rng.normal(size=4 * nf)
    link = rng.normal(size=(len(fib["n_nodes"]), 7))
    M = rng.normal(size=(3 * ns, 3 * ns)) / np.sqrt(3 * ns)
    with skb.Flow(0) as fl, skb.Dense(1) as dn:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])
        build(fl, prm)
        dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, M)
        res, v_s, v_b = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
        res_d, res_shell, v_b_d = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link, dense=dn)
        y = fl.apply_fiber_preconditioner(x)
        got = fl.get_fiber_operators()
        # the same operators uploaded instead of built: bitwise the same matvec and preconditioner
        fl.set_fiber_operators(got["A"], got["force"], got["xs"], prm["length_prev"], prm["plus_hinged"])
        fl.set_fiber_preconditioner(got["A_inv"])
        res2, v_s2, v_b2 = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
        res2_d, _, _ = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link, dense=dn)
        y2 = fl.apply_fiber_preconditioner(x)
        # and a build after an upload replaces it again; two builds are bitwise equal
        build(fl, prm)
        again = fl.get_fiber_operators()
        res3, _, _ = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
    ref_res, ref_v = orc.apply_matvec_fibers(fib, shell, body, ops, x, ETA, link)
    for r in (res, res_d):
        assert rel_max(r, ref_res) <= 1e-12 and rel_l2(r, ref_res) <= 1e-12
    assert rel_max(v_s, ref_v[nf:nf + ns]) <= 1e-12 and rel_max(v_b, ref_v[nf + ns:]) <= 1e-12
    assert rel_max(res_shell.reshape(-1), orc.periphery_dense_apply(M, shell["density"].reshape(-1),
                                                                    v_s.reshape(-1))) <= 1e-12
    assert np.array_equal(res, res2) and np.array_equal(v_s, v_s2) and np.array_equal(v_b, v_b2)
    assert np.array_equal(res_d, res2_d) and np.array_equal(y, y2) and np.array_equal(res, res3)
    for k in ("A", "force", "A_inv"):
        assert all(np.array_equal(a, b) for a, b in zip(got[k], again[k]))
    assert np.array_equal(got["xs"], again["xs"])


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_target_ranges_build_own_slice(system, world):
    from skellysim_b200.distributed import reference_rank_ranges
    fib, prm, _ = system
    shell, body = empty_shell_body(4, 90, 0)
    n_fibers, ns = len(fib["n_nodes"]), shell["pos"].shape[0]
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])
        build(fl, prm)
        full = fl.get_fiber_operators()
        off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
        for rank in range(world):
            f0, f1, s0, s1, b0, b1 = reference_rank_ranges(n_fibers, ns, 0, rank, world)
            fl.set_target_ranges(f0, f1, s0, s1, b0, b1)
            build(fl, prm, slice(f0, f1))
            own = fl.get_fiber_operators()
            for k in ("A", "force", "A_inv"):
                assert len(own[k]) == f1 - f0
                assert all(np.array_equal(a, b) for a, b in zip(own[k], full[k][f0:f1]))
            assert np.array_equal(own["xs"], full["xs"][off[f0]:off[f1]])


@pytest.mark.gpu
def test_multiflow_build(system):
    fib, prm, _ = system
    shell, body = empty_shell_body(5, 300, 0)
    rng = np.random.default_rng(6)
    nf = fib["pos"].shape[0]
    x = rng.normal(size=4 * nf)
    link = rng.normal(size=(len(fib["n_nodes"]), 7))
    args = [prm[k] for k in ("length_prev", "bending_rigidity", "radius", "penalty_param", "beta_tstep",
                             "minus_clamped", "plus_hinged")]
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])
        build(fl, prm)
        ref = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
    for devices in ([0, 0], [0, 0, 0]):
        with skb.MultiFlow(devices) as mf:
            mf.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
            mf.set_periphery(shell["pos"], shell["normals"])
            mf.set_bodies(body["pos"], body["normals"], body["centers"])
            for n in sorted(set(fib["n_nodes"])):
                m = fiber_fd.compute_matrices(n)
                mf.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
                mf.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
            mf.build_fiber_operators(*args, DT, ETA)
            res, o_s, v_b = mf.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
        assert rel_max(res, ref[0]) <= 1e-12 and rel_max(o_s, ref[1]) <= 1e-12, devices


@pytest.mark.gpu
def test_build_rejections():
    fib, prm = curved_fibers(12, [8, 16, 16])
    shell, body = empty_shell_body()
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        m8, m16 = fiber_fd.compute_matrices(8), fiber_fd.compute_matrices(16)
        fl.set_fiber_class(8, m8["D_1_0"], m8["P_downsample_bc"])
        fl.set_fiber_class_derivatives(8, m8["D_2_0"], m8["D_3_0"], m8["D_4_0"])
        with pytest.raises(skb.SkbError, match=r"fiber 1 has 16 nodes but skb_flow_set_fiber_class\("):
            build(fl, prm)
        fl.set_fiber_class(16, m16["D_1_0"], m16["P_downsample_bc"])
        with pytest.raises(skb.SkbError, match=r"fiber 1 has 16 nodes but skb_flow_set_fiber_class_derivatives"):
            build(fl, prm)
        fl.set_fiber_class_derivatives(16, m16["D_2_0"], m16["D_3_0"], m16["D_4_0"])
        build(fl, prm)
        for key, bad, pat in (("length_prev", 0.0, "fiber 2: length_prev"), ("radius", -1.0, "fiber 2: .*radius"),
                              ("minus_clamped", 2, "fiber 2: minus_clamped = 2"),
                              ("plus_hinged", -1, "fiber 2: .*plus_hinged = -1")):
            p = {k: np.array(v) for k, v in prm.items()}
            p[key][2] = bad
            with pytest.raises(skb.SkbError, match=pat):
                build(fl, p)
        with pytest.raises(skb.SkbError, match="dt = 0"):
            fl.build_fiber_operators(1.0, 1e-3, 1e-2, 500.0, 1.0, 0, 0, 0.0, ETA)
        with pytest.raises(skb.SkbError, match="eta = -1"):
            fl.build_fiber_operators(1.0, 1e-3, 1e-2, 500.0, 1.0, 0, 0, DT, -1.0)
        # a refused build leaves no operators behind
        with pytest.raises(skb.SkbError, match="set_fiber_operators"):
            fl.apply_fiber_force(np.zeros(4 * fib["pos"].shape[0]))
        with pytest.raises(skb.SkbError, match="8 <= n <= 128"):
            fl.set_fiber_class_derivatives(7, np.zeros((7, 7)), np.zeros((7, 7)), np.zeros((7, 7)))
    fib7, prm7 = curved_fibers(13, [7])
    with skb.Flow(0) as fl:
        load(fl, fib7, shell, body)
        fl.set_fiber_class(7, np.eye(7), np.zeros((14, 28)))  # (no 8-point stencil exists on 7 nodes)
        with pytest.raises(skb.SkbError, match="fiber 0 has 7 nodes: the device build takes 8 <= n <= 128"):
            build(fl, prm7)


@pytest.mark.gpu
def test_cpp_mirror_build(tmp_path):
    # tests/cpp/fiber_build_test.cpp: flow.hpp build -> read back -> upload round trip -> identical matvec; compiled here
    # against the in-tree headers and library
    here = os.path.dirname(os.path.abspath(__file__))
    root, libdir = os.path.dirname(here), os.path.dirname(skb.library_path())
    cxx = shutil.which("g++") or shutil.which("c++")
    assert cxx, "a C++ compiler is needed to build tests/cpp/fiber_build_test.cpp"
    exe = str(tmp_path / "fiber_build_test")
    subprocess.run([cxx, "-O2", "-std=c++17", "-Wall", "-I", os.path.join(root, "include"), "-o", exe,
                    os.path.join(here, "cpp", "fiber_build_test.cpp"), "-L", libdir, "-lskelly_b200",
                    f"-Wl,-rpath,{libdir}"], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr

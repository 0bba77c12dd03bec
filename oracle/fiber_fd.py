"""CPU restatement of FiberFiniteDifference's per-fiber matrices and operators -- TEST INFRASTRUCTURE ONLY (see
oracle/__init__.py: nothing under skellysim_b200/ may import this).

What the GPU path consumes as opaque dense arrays (SURVEY.md 8f N2) is produced here the way the reference produces
it, statement by statement, so that tests and bench.py run on operators with the reference's real structure
(`P_downsample_bc` block diagonal, derivative matrices banded, `A_` with its 14 boundary rows) instead of random
stand-ins.  Citations are `file:line` in the SkellySim tree:

    finite_diff               src/core/utils.cpp:48-102        (Fornberg's weights, sliding stencil of n_s points)
    barycentric_matrix        src/core/utils.cpp:12-36
    compute_matrices          src/core/fiber_finite_difference.cpp:519-558   (FiberFiniteDifference::matrices_)
    FiberOperators            src/core/fiber_finite_difference.cpp:62-72 (update_derivatives), :97-187
                              (update_linear_operator), :317-335 (update_force_operator), :347-516
                              (apply_bc_rectangular), include/fiber_finite_difference.hpp:140-144 (update_constants)

PARITY STATUS.  The reference's fiber code needs Eigen / toml11 / spdlog / MPI and cannot be compiled here, it has no
Python twin, and its unit test (tests/core/unit_tests/unit_test_fiber_finite_difference.cpp) stores no numbers -- so
nothing of the reference can run against this file.  What IS pinned (tests/test_oracle_fiber_fd.py): `weights_0` and the
block layout of `P_downsample_bc` against the literal statements :545-555; `finite_diff` is exact on polynomials up to
the stencil's degree and `barycentric_matrix` reproduces polynomials (the properties Fornberg's and Berrut-Trefethen's
formulas are defined by); `FiberOperators` annihilates what it must (a straight fiber has xss = 0, force_operator_ of a
uniform tension...).  The remaining risk is a shared misreading of update_linear_operator / apply_bc_rectangular's
coefficients; the GPU kernels do not depend on those values (they are dense GEMV operands).
"""
from __future__ import annotations

import numpy as np

ALLOWED_N_NODES = (8, 16, 24, 32, 48, 64, 96, 128)  # fiber_finite_difference.cpp:522


def finite_diff(s, M: int, n_s: int):
    """utils::finite_diff (utils.cpp:48-102): M-th derivative matrix on the grid s with an n_s-point sliding stencil
    (one-sided near the ends)."""
    s = np.asarray(s, dtype=np.float64)
    size = s.shape[0]
    D = np.zeros((size, size))
    n_s_half = (n_s - 1) // 2                                     # :51
    n_s = n_s - 1                                                 # :52
    for xi in range(size):
        si = s[xi]
        if xi < n_s_half:                                         # :58-60
            xlow, xhigh = 0, n_s + 1
        elif xi > (size - n_s_half - 2):                          # :61-63
            xlow, xhigh = -n_s - 1, size
        else:                                                     # :64-67
            xlow, xhigh = xi - n_s_half, xi - n_s_half + n_s + 1
        if xlow < 0:                                              # :68
            xlow = size + xlow
        x = s[xlow:xhigh]
        c1 = 1.0
        c4 = x[0] - si
        c = np.zeros((n_s + 1, M + 1))
        c[0, 0] = 1.0
        for i in range(1, n_s + 1):                               # :78-98
            mn = min(i, M)
            c2 = 1.0
            c5 = c4
            c4 = x[i] - si
            for j in range(i):
                c3 = x[i] - x[j]
                c2 = c2 * c3
                if j == i - 1:
                    for k in range(mn, 0, -1):
                        c[i, k] = c1 * (k * c[i - 1, k - 1] - c5 * c[i - 1, k]) / c2
                    c[i, 0] = -c1 * c5 * c[i - 1, 0] / c2
                for k in range(mn, 0, -1):
                    c[j, k] = (c4 * c[j, k] - k * c[j, k - 1]) / c3
                c[j, 0] = c4 * c[j, 0] / c3
            c1 = c2
        for i in range(n_s + 1):                                  # :99-101
            D[xi, xlow + i] = c[i, M]
    return D


def barycentric_matrix(x, y):
    """utils::barycentric_matrix (utils.cpp:12-36): resampling matrix from the N points x to the M points y."""
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    N, M = x.shape[0], y.shape[0]
    w = np.ones(N)
    w[1::2] = -1.0                                                # :17-18
    w[0] = 0.5                                                    # :19
    w[N - 1] = -0.5 * (-1.0) ** N                                 # :20
    P = np.zeros((M, N))
    eps = np.finfo(np.float64).eps
    for j in range(M):
        with np.errstate(divide="ignore"):
            S = float(np.sum(w / (y[j] - x)))                     # :24-27
        for k in range(N):
            if abs(y[j] - x[k]) > eps:                            # :29-32
                P[j, k] = w[k] / (y[j] - x[k]) / S
            else:
                P[j, k] = 1.0
    return P


_MATRICES = {}


def compute_matrices(n_nodes: int, n_nodes_finite_diff: int = 4):
    """One entry of FiberFiniteDifference::matrices_ (fiber_finite_difference.cpp:519-562; the reference builds it with
    n_nodes_finite_diff = 4).  Returns a dict with the reference's member names; D_k_0 are stored PRE-TRANSPOSED exactly
    like the reference does (:537-540)."""
    key = (n_nodes, n_nodes_finite_diff)
    if key in _MATRICES:
        return _MATRICES[key]
    n = int(n_nodes)
    alpha = np.linspace(-1.0, 1.0, n)                                                     # :524
    n_roots = n - 4                                                                       # :526
    alpha_roots = 2 * (0.5 + np.linspace(0, n_roots - 1, n_roots)) / n_roots - 1          # :527
    n_tension = n - 2                                                                     # :529
    alpha_tension = 2 * (0.5 + np.linspace(0, n_tension - 1, n_tension)) / n_tension - 1  # :530-531
    m = dict(alpha=alpha, alpha_roots=alpha_roots, alpha_tension=alpha_tension)
    for k in (1, 2, 3, 4):                                                                # :537-540
        m[f"D_{k}_0"] = finite_diff(alpha, k, n_nodes_finite_diff + k).T.copy()
    m["P_X"] = barycentric_matrix(alpha, alpha_roots)                                     # :542
    m["P_T"] = barycentric_matrix(alpha, alpha_tension)                                   # :543
    w = np.ones(n) * 2.0                                                                  # :545-548
    w[0] = w[-1] = 1.0
    m["weights_0"] = w / (n - 1)
    P = np.zeros((4 * n - 14, 4 * n))                                                     # :551-555
    P[0 * (n - 4):1 * (n - 4), 0 * n:1 * n] = m["P_X"]
    P[1 * (n - 4):2 * (n - 4), 1 * n:2 * n] = m["P_X"]
    P[2 * (n - 4):3 * (n - 4), 2 * n:3 * n] = m["P_X"]
    P[3 * (n - 4):3 * (n - 4) + (n - 2), 3 * n:4 * n] = m["P_T"]
    m["P_downsample_bc"] = P
    _MATRICES[key] = m
    return m


BC_FORCE, BC_TORQUE, BC_VELOCITY, BC_ANGULAR_VELOCITY = "Force", "Torque", "Velocity", "AngularVelocity"


class FiberOperators:
    """The per-timestep operators of ONE FiberFiniteDifference, built as System::prep_state_for_solver does:
    update_derivatives -> update_linear_operator -> apply_bc_rectangular -> update_force_operator (-> A_LU_).

    x: (n, 3) node positions (the reference's 3 x n, column-major); free fiber by default (bc Force/Torque both ends,
    fiber_finite_difference.cpp:74-95); minus_clamped / plus_pinned select the other branches."""

    def __init__(self, x, length, bending_rigidity=2.5e-3, radius=0.0125, eta=1.0, dt=1e-2, length_prev=None,
                 minus_clamped=False, plus_pinned=False, penalty_param=500.0, beta_tstep=1.0, dtype=np.float64,
                 absolute=False):
        """dtype: the arithmetic.  The inputs (positions, scalars, the class matrices of compute_matrices) are float64
        values either way, so np.longdouble evaluates exactly the function of them that a float64 evaluation rounds.

        absolute=True evaluates the error scale S of every output instead: the same computation with every input
        replaced by |.| and every subtraction turned into an addition (c_0 = -log(e eps^2) / (8 pi eta) enters as
        (|log(e eps^2)| + 4) / (8 pi eta): the log's absolute error is u times that).  Any float64 evaluation order of
        an output y then satisfies |fl(y) - y| <= gamma_k S(y), k the operations on its longest path."""
        f = np.dtype(dtype).type
        x = np.asarray(x, dtype=np.float64).astype(f)
        self.n = n = x.shape[0]
        self.x = np.abs(x) if absolute else x
        self.sg = f(1.0 if absolute else -1.0)                            # the sign of every subtraction
        self.dtype = f
        self.length = f(np.float64(length))
        self.length_prev = f(np.float64(length if length_prev is None else length_prev))
        self.E = f(np.float64(bending_rigidity))
        eta = f(np.float64(eta))
        eps = f(np.float64(radius)) / self.length                         # fiber_finite_difference.hpp:141
        lg = np.log(f(np.e) * eps ** 2)
        self.c_0 = (np.abs(lg) + 4) / (8 * f(np.pi) * eta) if absolute else -lg / (8 * f(np.pi) * eta)   # :142
        self.c_1 = 2.0 / (8.0 * f(np.pi) * eta)                           # :143
        self.penalty, self.beta, self.dt = (f(np.float64(v)) for v in (penalty_param, beta_tstep, dt))
        self.bc_minus = (BC_VELOCITY, BC_ANGULAR_VELOCITY) if minus_clamped else (BC_FORCE, BC_TORQUE)   # :75-78
        self.bc_plus = (BC_VELOCITY, BC_TORQUE) if plus_pinned else (BC_FORCE, BC_TORQUE)               # :84-88
        self.mats = compute_matrices(n)
        self._m = {k: (np.abs(v) if absolute else v).astype(f) for k, v in self.mats.items()
                   if k.startswith("D_") or k == "P_downsample_bc"}
        self._update_derivatives()
        self._update_linear_operator()
        self._apply_bc_rectangular()
        self._update_force_operator()

    # xs_ = (2/L_prev)^k * x_ * D_k_0 with x_ 3 x n  ==  (n,3): D_k_0^T-free form x^T-consistent: (x_ D)^T = D^T x
    def _update_derivatives(self):                                        # fiber_finite_difference.cpp:62-72
        m, x, lp = self._m, self.x, self.length_prev
        self.xs = (2.0 / lp) ** 1 * (m["D_1_0"].T @ x)
        self.xss = (2.0 / lp) ** 2 * (m["D_2_0"].T @ x)
        self.xsss = (2.0 / lp) ** 3 * (m["D_3_0"].T @ x)
        self.xssss = (2.0 / lp) ** 4 * (m["D_4_0"].T @ x)

    def _update_linear_operator(self):                                    # :97-187
        n, m, L, sg = self.n, self._m, self.length, self.sg
        D_1 = m["D_1_0"].T * (2.0 / L) ** 1                               # :101-104
        D_2 = m["D_2_0"].T * (2.0 / L) ** 2
        D_3 = m["D_3_0"].T * (2.0 / L) ** 3
        D_4 = m["D_4_0"].T * (2.0 / L) ** 4
        E, c0, c1 = self.E, self.c_0, self.c_1
        xs, xss, xsss = self.xs, self.xss, self.xsss
        I = np.eye(n, dtype=self.dtype)
        cw = lambda D, v: D * v[:, None]                                  # (D.colwise() * v): row i scaled by v_i
        A = np.zeros((4 * n, 4 * n), dtype=self.dtype)
        blk = lambda r, c: (slice(r * n, (r + 1) * n), slice(c * n, (c + 1) * n))
        for a in range(3):                                                # :146-159
            for b in range(3):
                if a == b:
                    A[blk(a, a)] = (self.beta / self.dt * I + E * c0 * cw(D_4, 1.0 + xs[:, a] ** 2)
                                    + E * c1 * cw(D_4, 1.0 + sg * xs[:, a] ** 2))
                else:
                    A[blk(a, b)] = E * (c0 + sg * c1) * cw(D_4, xs[:, a] * xs[:, b])
            A[blk(a, 3)] = sg * (c0 * 2.0) * cw(D_1, xs[:, a]) + sg * (c0 + c1) * np.diag(xss[:, a])      # :161-168
            A[blk(3, a)] = (sg * (c1 + 7.0 * c0) * E * cw(D_4, xss[:, a]) + sg * 6.0 * c0 * E * cw(D_3, xsss[:, a])
                            + sg * self.penalty * cw(D_1, xs[:, a]))                                   # :173-183
        A[blk(3, 3)] = sg * 2.0 * c0 * D_2 + (c0 + c1) * np.diag(np.sum(xss ** 2, axis=1))             # :185-186
        self.A = A

    def _apply_bc_rectangular(self):                                      # :347-516 (operator part; RHS not needed)
        n, m, L, sg = self.n, self._m, self.length, self.sg
        D_1 = m["D_1_0"].T * (2.0 / L) ** 1
        D_2 = m["D_2_0"].T * (2.0 / L) ** 2
        D_3 = m["D_3_0"].T * (2.0 / L) ** 3
        E, c0 = self.E, self.c_0
        xs, xss = self.xs, self.xss
        A = self.A
        A[:4 * n - 14] = m["P_downsample_bc"] @ A                         # :356
        B = np.zeros((14, 4 * n), dtype=self.dtype)                                       # :362-363
        bdt = self.beta / self.dt
        if self.bc_minus[0] == BC_VELOCITY:                               # :366-384
            B[0, 0 * n] = B[1, 1 * n] = B[2, 2 * n] = bdt
            for k in range(3):
                B[3, k * n:(k + 1) * n] = (6.0 * E * c0) * xss[0, k] * D_3[0]
            B[3, 3 * n:4 * n] = (2.0 * c0) * D_1[0]
        else:                                                             # Force :386-405
            for k in range(3):
                B[k, k * n:(k + 1) * n] = E * D_3[0]
                B[k, 3 * n] = sg * xs[0, k]
                B[3, k * n:(k + 1) * n] = sg * E * D_2[0] * xss[0, k]
            B[3, 3 * n] = sg
        if self.bc_minus[1] == BC_ANGULAR_VELOCITY:                       # :415-424
            for k in range(3):
                B[4 + k, k * n:(k + 1) * n] = bdt * D_1[0]
        else:                                                             # Torque :426-433
            for k in range(3):
                B[4 + k, k * n:(k + 1) * n] = D_2[0]
        e = n - 1
        if self.bc_plus[0] == BC_VELOCITY:                                # :443-464
            B[7, 1 * n - 1] = B[8, 2 * n - 1] = B[9, 3 * n - 1] = bdt
            for k in range(3):
                B[10, k * n:(k + 1) * n] = (6.0 * E * c0) * D_3[e] * xss[e, k]
            B[10, 3 * n:4 * n] = (2.0 * c0) * D_1[e]
        else:                                                             # Force :466-487
            for k in range(3):
                B[7 + k, k * n:(k + 1) * n] = sg * E * D_3[e]
                B[7 + k, 4 * n - 1] = xs[e, k]
                B[10, k * n:(k + 1) * n] = E * D_2[e] * xss[e, k]
            B[10, 4 * n - 1] = 1.0
        for k in range(3):                                                # plus Torque :497-505
            B[11 + k, k * n:(k + 1) * n] = D_2[e]
        A[4 * n - 14:] = B
        self.A = A

    def _update_force_operator(self):                                     # :317-335
        n, m, L, sg = self.n, self._m, self.length, self.sg
        D_1 = m["D_1_0"] * (2.0 / L) ** 1
        D_4 = m["D_4_0"] * (2.0 / L) ** 4
        F = np.zeros((3 * n, 4 * n), dtype=self.dtype)
        for i in range(3):
            F[i * n:(i + 1) * n, i * n:(i + 1) * n] = self.sg * self.E * D_4.T                                  # :328
            blk = np.diag(self.xss[:, i])                                                               # :330
            blk = blk + (D_1 * self.xs[:, i][None, :]).T                                                # :332-333
            F[i * n:(i + 1) * n, 3 * n:4 * n] = blk
        self.force_operator = F

    @property
    def plus_bc_velocity(self) -> int:
        return int(self.bc_plus[0] == BC_VELOCITY)


def suspension_operators(r_fib, n_nodes, lengths, eta=1.0, dt=1e-2, seed=0, clamp_fraction=0.0, pin_fraction=0.0):
    """Operators of a whole fiber container in the layout the device API takes (oracle.fiber_container_matvec's `ops`
    dict): A / force lists, xs (N_f,3), length_prev, plus, D_1_0 / P per node count."""
    rng = np.random.default_rng(seed)
    ops = dict(n_nodes=[int(n) for n in n_nodes], A=[], force=[], D_1_0={}, P={}, length_prev=[], plus=[])
    xs, off = [], 0
    for n, L in zip(ops["n_nodes"], lengths):
        fo = FiberOperators(np.asarray(r_fib)[off:off + n], L, eta=eta, dt=dt,
                            minus_clamped=bool(rng.random() < clamp_fraction),
                            plus_pinned=bool(rng.random() < pin_fraction))
        ops["A"].append(fo.A)
        ops["force"].append(fo.force_operator)
        xs.append(fo.xs)
        ops["length_prev"].append(fo.length_prev)
        ops["plus"].append(fo.plus_bc_velocity)
        if n not in ops["D_1_0"]:
            ops["D_1_0"][n] = fo.mats["D_1_0"]
            ops["P"][n] = fo.mats["P_downsample_bc"]
        off += n
    ops["xs"] = np.concatenate(xs) if xs else np.zeros((0, 3))
    return ops


def gauss_jordan_inverse(A, dtype=np.float64, pivot_window=None, pivoting=True, recip_rel_err=0.0):
    """Host restatement of fiber_build.cuh's fiber_inverse_kernel in `dtype`: in-place Gauss-Jordan elimination with
    partial pivoting (the first row of largest magnitude in rows [k, m)), the pivot row scaled by the reciprocal of the
    pivot, column k eliminated from every other row with the pivot column as it was before the step, and the column
    interchanges that undo the pivoting applied at the end as one permutation.  The kernel fuses the elimination's
    multiply-add; numpy rounds the product first.  np.longdouble gives the extended-precision inverse of the same
    float64 matrix.

    The keyword arguments plant defects that a test of the kernel must catch: a pivot search over rows [k, k +
    pivot_window) only, no pivoting at all, a pivot reciprocal off by the relative error recip_rel_err."""
    M = np.array(A, dtype=np.float64).astype(dtype)
    m = M.shape[0]
    piv = np.empty(m, dtype=np.int64)
    for k in range(m):
        p = k
        if pivoting:
            hi = m if pivot_window is None else min(m, k + pivot_window)
            p = k + int(np.argmax(np.abs(M[k:hi, k])))
        piv[k] = p
        rc = M[:, k].copy()                              # the published pivot column, row-swapped
        rc[k], rc[p] = rc[p], rc[k]
        if p != k:
            M[[k, p]] = M[[p, k]]
        inv = 1 / rc[k]
        if recip_rel_err:
            inv = inv * (1 + recip_rel_err)
        r = M[k] * inv
        r[k] = inv
        M[k] = r
        M[:k, k] = 0
        M[k + 1:, k] = 0
        M[:k] -= np.outer(rc[:k], r)
        M[k + 1:] -= np.outer(rc[k + 1:], r)
    perm = np.arange(m)
    for k in range(m - 1, -1, -1):
        perm[k], perm[piv[k]] = perm[piv[k]], perm[k]
    return M[:, perm]


def extended_inverse(A):
    """A^-1 of the float64 matrix A in np.longdouble: Gauss-Jordan with partial pivoting and one step of iterative
    refinement with a long-double residual, X <- X + X (I - A X).  Also returns the correction a second step would
    apply, an independent estimate of the extended inverse's own error."""
    if np.finfo(np.longdouble).nmant < 63:
        raise RuntimeError(f"np.longdouble has {np.finfo(np.longdouble).nmant + 1} mantissa bits here; an extended-"
                           "precision reference needs at least 64")
    A_ext = np.asarray(A, dtype=np.float64).astype(np.longdouble)
    I = np.eye(A_ext.shape[0], dtype=np.longdouble)
    X = gauss_jordan_inverse(A, np.longdouble)
    X = X + X @ (I - A_ext @ X)
    return X, X @ (I - A_ext @ X)

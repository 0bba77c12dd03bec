"""CPU tests of tests/gmres_reference.py, the host restatement of skb_flow_solve_system: its iterates are those of GMRES
written as a least-squares problem over an explicitly built Krylov space, with and without restarts; its edge cases
behave as specified; and each planted defect is caught."""
import numpy as np
import pytest

import gmres_reference as gr


def system(n, seed, spread=0.3):
    """a random nonsymmetric well-conditioned A = I + spread G / sqrt(n) and a preconditioner P^-1 = inverse of a
    perturbed A (so A P^-1 is near but not at I)"""
    rng = np.random.default_rng(seed)
    A = np.eye(n) + spread * rng.normal(size=(n, n)) / np.sqrt(n)
    P = A + 0.2 * rng.normal(size=(n, n)) / np.sqrt(n)
    Pinv = np.linalg.inv(P)
    return A, Pinv, rng.normal(size=n)


def krylov_minimizer(A, Pinv, r, k):
    """z = argmin ||r - A P^-1 z|| over K_k(A P^-1, r), built explicitly (QR of [r, AP r, ...]); returns P^-1 z"""
    AP = A @ Pinv
    K = [r]
    for _ in range(k - 1):
        K.append(AP @ K[-1])
    Q, _ = np.linalg.qr(np.stack(K, axis=1))
    c = np.linalg.lstsq(AP @ Q, r, rcond=None)[0]
    return Pinv @ (Q @ c)


def run(A, Pinv, b, **kw):
    return gr.gmres(lambda v: A @ v, lambda v: Pinv @ v, b, **kw)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_iterates_without_restarts_are_the_krylov_minimizers(seed):
    A, Pinv, b = system(60, seed)
    for k in (1, 3, 7, 12):
        x, info = run(A, Pinv, b, tol=1e-300, num_blocks=50, max_iters=k)
        assert info["iterations"] == k and info["restarts"] == 0 and not info["converged"]
        ref = krylov_minimizer(A, Pinv, b, k)
        assert np.linalg.norm(x - ref) <= 1e-11 * np.linalg.norm(ref), k
        # the implicit estimate is the true residual of the iterate
        assert abs(info["history"][k] - np.linalg.norm(b - A @ x) / np.linalg.norm(b)) <= 1e-12


@pytest.mark.parametrize("m", [3, 5])
def test_restarted_iterates_are_gmres_m_cycle_by_cycle(m):
    A, Pinv, b = system(50, 7, spread=0.6)
    x_ref = np.zeros_like(b)
    for cycle in range(1, 5):
        x_ref = x_ref + krylov_minimizer(A, Pinv, b - A @ x_ref, m)
        x, info = run(A, Pinv, b, tol=1e-300, num_blocks=m, max_iters=cycle * m)
        assert info["iterations"] == cycle * m and info["restarts"] == cycle - 1
        assert np.linalg.norm(x - x_ref) <= 1e-11 * np.linalg.norm(x_ref), cycle


@pytest.mark.parametrize("r", [1, 2, 5])
def test_identity_plus_rank_r_converges_in_r_plus_1_steps(r):
    """The Krylov space of I + rank r has dimension <= r + 1: step r + 1 finds no new direction.  In floating point its
    new vector is either below the breakdown threshold or so small that the implicit estimate ends the cycle; both
    paths end it there, and the explicit check holds"""
    rng = np.random.default_rng(10 + r)
    n = 40
    A = np.eye(n) + rng.normal(size=(n, r)) @ rng.normal(size=(r, n)) / n
    b = rng.normal(size=n)
    x, info = run(A, np.eye(n), b, tol=1e-15, num_blocks=30, max_iters=100)
    assert info["converged"] and info["iterations"] <= r + 1, info
    assert np.linalg.norm(b - A @ x) <= 1e-15 * np.linalg.norm(b)


@pytest.mark.parametrize("n", [10, 50])
def test_an_invariant_krylov_space_is_an_exact_solve(n):
    """b in a two-dimensional invariant subspace of A: the second step's new vector vanishes to rounding, the breakdown
    path takes it as an exact solve, and the explicit check confirms it"""
    A = np.diag(np.r_[np.full(n - 1, 2.0), 3.0])
    b = np.zeros(n)
    b[[0, 3, n - 1]] = 1.0, 0.2, 0.7
    x, info = run(A, np.eye(n), b, tol=1e-14, num_blocks=30, max_iters=30)
    assert info["converged"] and info["iterations"] == 2 and info["breakdowns"] == 1, info
    assert info["history"][-1] == 0.0
    assert np.linalg.norm(b - A @ x) <= 1e-14 * np.linalg.norm(b)


def test_zero_rhs_gives_zero_in_zero_steps():
    A, Pinv, _ = system(20, 3)
    x, info = run(A, Pinv, np.zeros(20))
    assert np.array_equal(x, np.zeros(20)) and info["converged"] and info["iterations"] == 0
    assert info["residual"] == 0.0 and list(info["history"]) == [0.0]


def test_max_iters_returns_the_current_iterate_unconverged():
    A, Pinv, b = system(80, 4, spread=1.5)
    x, info = run(A, Pinv, b, tol=1e-12, num_blocks=10, max_iters=6)
    assert not info["converged"] and info["iterations"] == 6
    assert np.allclose(x, krylov_minimizer(A, Pinv, b, 6), rtol=0, atol=1e-11 * np.linalg.norm(x))
    assert info["residual"] == pytest.approx(np.linalg.norm(b - A @ x), rel=1e-12)
    x0, info0 = run(A, Pinv, b, max_iters=0)
    assert np.array_equal(x0, np.zeros_like(b)) and not info0["converged"] and info0["explicit_residual"] == 1.0


@pytest.mark.parametrize("seed,m", [(s, m) for s in range(4) for m in (4, 300)])
def test_every_convergence_meets_the_explicit_check(seed, m):
    A, Pinv, b = system(70, 20 + seed, spread=1.0)
    tol = 1e-10
    x, info = run(A, Pinv, b, tol=tol, num_blocks=m, max_iters=1000)
    assert info["converged"]
    assert np.linalg.norm(b - A @ x) <= tol * np.linalg.norm(b)
    assert info["explicit_residual"] <= tol and info["history"][-1] <= tol


def test_left_preconditioning_misses_the_explicit_residual():
    rng = np.random.default_rng(30)
    n = 60
    A = np.eye(n) + 0.3 * rng.normal(size=(n, n)) / np.sqrt(n)
    Pinv = np.diag(np.logspace(-4, 0, n))  # badly scaled: ||P^-1 r|| says little about ||r||
    b = rng.normal(size=n)
    tol = 1e-8
    x, info = run(A, Pinv, b, tol=tol, max_iters=200)
    assert info["converged"] and np.linalg.norm(b - A @ x) <= tol * np.linalg.norm(b)
    xl, infol = run(A, Pinv, b, tol=tol, max_iters=200, defect="left")
    assert infol["converged"] and np.linalg.norm(b - A @ xl) > tol * np.linalg.norm(b)


def test_dropping_p_inv_from_the_update_is_caught():
    """the first cycle's implicit estimate meets tol, its explicit residual does not: the defect restarts again and
    again where the correct update converges in one cycle"""
    A, Pinv, b = system(60, 31)
    x, ok = run(A, Pinv, b, tol=1e-10, max_iters=200)
    assert ok["converged"] and ok["restarts"] == 0
    _, info = run(A, Pinv, b, tol=1e-10, max_iters=200, defect="no_pinv")
    assert info["restarts"] >= 5 and info["iterations"] > 5 * ok["iterations"], info


def test_one_gram_schmidt_pass_loses_orthogonality():
    """A Krylov sequence that loses orthogonality under classical Gram-Schmidt: A with eigenvalues spread over
    sixteen decades, so the Krylov vectors align quickly with the dominant eigenvectors"""
    rng = np.random.default_rng(32)
    n = 80
    Q, _ = np.linalg.qr(rng.normal(size=(n, n)))
    A = Q @ np.diag(np.logspace(0, 16, n)) @ Q.T
    b = rng.normal(size=n)
    kw = dict(tol=1e-300, num_blocks=40, max_iters=40, keep_basis=True)
    _, info = run(A, np.eye(n), b, **kw)
    _, bad = run(A, np.eye(n), b, defect="one_pass", **kw)
    lost = lambda V: np.abs(V.T @ V - np.eye(V.shape[1])).max()
    assert lost(info["basis"]) <= 1e-12, lost(info["basis"])
    assert lost(bad["basis"]) > 1e-8, lost(bad["basis"])


def test_a_flipped_givens_sign_is_caught():
    A, Pinv, b = system(60, 33)
    for k in (3, 8):
        x, _ = run(A, Pinv, b, tol=1e-300, num_blocks=50, max_iters=k, defect="givens")
        ref = krylov_minimizer(A, Pinv, b, k)
        assert np.linalg.norm(x - ref) > 1e-6 * np.linalg.norm(ref)


def test_blocked_dot_is_a_dot():
    rng = np.random.default_rng(34)
    for n in (1, 31, 33, 1000, 20001):
        V, w = rng.normal(size=(n, 5)), rng.normal(size=n)
        assert np.allclose(gr.blocked_dot(V, w), V.T @ w, rtol=1e-13, atol=1e-13 * np.sqrt(n))

"""Host restatement of skb_flow_solve_system (skellysim_b200/csrc/skb_solve.cu): Solver::solve (solver_hydro.cpp:64-95)
as the reference configures Belos -- restarted GMRES, right preconditioning, x0 = 0, ICGS (two classical Gram-Schmidt
passes), Givens rotations, the implicit estimate ending a cycle and the explicit ||b - A x|| deciding convergence.
numpy, float64, step for step as the device solve, with A and P^-1 as callables.

`dot(V, w)` computes V^T w (V a 2-D array of columns); numpy's by default, or `blocked_dot` for the device kernels'
summation order.  `defect` plants one error, for the tests that show each is caught:
  "left"       left instead of right preconditioning (GMRES on P^-1 A, P^-1 b; the checks on the preconditioned residual)
  "no_pinv"    P^-1 dropped from the cycle-end update (x += V y)
  "one_pass"   one classical Gram-Schmidt pass instead of two
  "givens"     the sign of the Givens rotation's s flipped where it is applied to g
"""
import numpy as np

BREAKDOWN = 16.0 * 2.0 ** -53  # a new vector at most this fraction of its norm before ICGS spans nothing new


def blocked_dot(V, w, ctas=528, tile=32, warps=8):
    """V^T w summed as krylov_pass_kernel and krylov_combine_kernel sum it: per row block (one per CTA, rows rounded to
    whole tiles) the tiles in order, inside a tile a shuffle tree over 32 lanes; then the blocks: 128 strided running
    sums combined by a tree"""
    n = w.shape[0]
    V = V.reshape(n, -1)
    ctas0 = max(1, min(ctas, -(-n // tile)))
    rows_per = -(-(-(-n // ctas0)) // tile) * tile
    parts = []
    for r0 in range(0, n, rows_per):
        acc = np.zeros(V.shape[1])
        for t0 in range(r0, min(n, r0 + rows_per), tile):
            t1 = min(n, r0 + rows_per, t0 + tile)
            p = np.zeros((tile, V.shape[1]))
            p[:t1 - t0] = V[t0:t1] * w[t0:t1, None]
            for o in (16, 8, 4, 2, 1):
                p[:o] = p[:o] + p[o:2 * o]
            acc = acc + p[0]
        parts.append(acc)
    parts = np.array(parts)
    lanes = np.zeros((128, V.shape[1]))
    for c in range(parts.shape[0]):
        lanes[c % 128] = lanes[c % 128] + parts[c]
    h = 64
    while h:
        lanes[:h] = lanes[:h] + lanes[h:2 * h]
        h //= 2
    return lanes[0]


def _np_dot(V, w):
    return V.T @ w


def gmres(A, P_inv, b, tol=1e-10, num_blocks=300, max_iters=1000, dot=_np_dot, defect=None, keep_basis=False):
    """x = A^-1 b.  Returns (x, info): info has converged, iterations, restarts, implicit_residual, explicit_residual,
    residual (as skb_solve_info), history (the implicit relative residual after each step, history[0] = 1), breakdowns,
    and with keep_basis the basis of the last cycle (n x (k + 1))."""
    b = np.asarray(b, dtype=np.float64)
    n, m = b.shape[0], int(num_blocks)
    left = defect == "left"
    Op = (lambda v: P_inv(A(v))) if left else (lambda v: A(P_inv(v)))
    rhs = P_inv(b) if left else b
    norm = lambda v: np.sqrt(dot(v[:, None], v)[0])
    x = np.zeros(n)
    r = rhs.copy()
    bnorm = norm(r)
    target = tol * bnorm
    beta = est = bnorm
    info = dict(converged=0, iterations=0, restarts=0, breakdowns=0, history=[1.0 if bnorm > 0 else 0.0])
    total = 0
    converged = beta <= target
    basis = None
    while not converged and total < max_iters:
        V = np.zeros((n, m + 1))
        V[:, 0] = r / beta
        H = np.zeros((m + 1, m))
        cs, sn, g = np.zeros(m), np.zeros(m), np.zeros(m + 1)
        g[0] = beta
        k = 0
        while k < m and total < max_iters:
            w = Op(V[:, k])
            h1 = dot(V[:, :k + 1], w)
            w0 = norm(w)
            w = w - V[:, :k + 1] @ h1
            if defect == "one_pass":
                h = h1
            else:
                h2 = dot(V[:, :k + 1], w)
                w = w - V[:, :k + 1] @ h2
                h = h1 + h2
            bet = norm(w)
            breakdown = not bet > BREAKDOWN * w0
            if breakdown:
                bet = 0.0
                info["breakdowns"] += 1
            col = np.zeros(m + 1)
            col[:k + 1] = h
            col[k + 1] = bet
            for i in range(k):
                t = cs[i] * col[i] + sn[i] * col[i + 1]
                col[i + 1] = -sn[i] * col[i] + cs[i] * col[i + 1]
                col[i] = t
            rr = np.hypot(col[k], col[k + 1])
            cs[k], sn[k] = (col[k] / rr, col[k + 1] / rr) if rr > 0 else (1.0, 0.0)
            col[k], col[k + 1] = rr, 0.0
            H[:, k] = col
            g[k + 1] = (sn[k] if defect == "givens" else -sn[k]) * g[k]
            g[k] = cs[k] * g[k]
            k += 1
            total += 1
            est = abs(g[k])
            info["history"].append(est / bnorm)
            if breakdown or est <= target:
                break
            V[:, k] = w / bet
        kk = 0
        while kk < k and H[kk, kk] != 0.0:
            kk += 1
        y = np.zeros(kk)
        for i in range(kk - 1, -1, -1):
            y[i] = (g[i] - H[i, i + 1:kk] @ y[i + 1:kk]) / H[i, i]
        if kk:
            u = V[:, :kk] @ y
            x = x + (u if left or defect == "no_pinv" else P_inv(u))
        r = (P_inv(b - A(x)) if left else b - A(x))
        beta = norm(r)
        converged = beta <= target
        if not converged and total < max_iters:
            info["restarts"] += 1
        if keep_basis:
            basis = V[:, :k + 1]
    info.update(converged=int(converged), iterations=total, implicit_residual=est / bnorm if bnorm > 0 else 0.0,
                explicit_residual=beta / bnorm if bnorm > 0 else 0.0, residual=beta,
                history=np.array(info["history"]))
    if keep_basis:
        info["basis"] = basis
    return x, info

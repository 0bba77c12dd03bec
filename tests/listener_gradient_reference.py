"""numpy restatement, in long double, of skb_flow_listener_gradient: the analytic velocity gradient and pressure of every
source of the listener's velocity (System::velocity_at_targets), with the body-interior rule.

Conventions: r = x_trg - x_src, c = 1 / (8 pi eta); G[t, i, j] = d u_i / d x_j at target t; a coincident pair (r == 0)
adds exactly 0 to every output; the pressure goes to 0 far from every source.
  Stokeslet  u_i = c (f_i / r + r_i (f.r) / r^3):
             G_ij = c ((delta_ij (f.r) - f_i r_j + r_i f_j) / r^3 - 3 r_i r_j (f.r) / r^5),  p = (f.r) / (4 pi r^3)
  stresslet  u = kappa r (r.S.r) / r^5, kappa = -3 / (8 pi eta), S = 2 eta n (x) rho (the library's scaling):
             G_ij = kappa (delta_ij A + r_i ((S + S^T) r)_j - 5 r_i r_j A / r^2) / r^5,  A = r.S.r,
             p = 2 kappa eta (A - tr(S) r^2 / 3) / r^5
  rotlet     u = c (L x r) / D^3: G_ij = c (eps_iaj L_a / D^3 - 3 (L x r)_i r_j / D^5), no pressure
  Oseen      u = c (f / D + r (r.f) / D^3): the Stokeslet's G and p with D for r
  with D = sqrt(r^2 + reg^2) in the regularised branch of the velocity kernel (rotlet: r^2 < eps^2; Oseen: r <= eps),
  else r, and dD / dr_j = r_j / D in both branches.
"""
import numpy as np

LD = np.longdouble
PI = LD("3.14159265358979323846264338327950288")
REG, EPS = 5e-3, 1e-5
_CHUNK = 1 << 17  # (target, source) pairs per block


def _ld(x, cols):
    return np.asarray(x, dtype=LD).reshape(-1, cols)


def _blocks(n_trg, n_src):
    step = max(1, _CHUNK // max(n_src, 1))
    for a in range(0, n_trg, step):
        yield slice(a, min(n_trg, a + step))


def _pairs(r_src, r_trg, sl):
    d = r_trg[sl, None, :] - r_src[None, :, :]
    r2 = np.einsum("tsk,tsk->ts", d, d)
    return d, r2


def stokeslet(r_src, f, r_trg, eta):
    """(G (n, 3, 3), p (n,)) of plain Stokeslets f at r_src"""
    r_src, f, r_trg = _ld(r_src, 3), _ld(f, 3), _ld(r_trg, 3)
    eta = LD(eta)
    G, p = np.zeros((len(r_trg), 3, 3), dtype=LD), np.zeros(len(r_trg), dtype=LD)
    if len(r_src) == 0:
        return G, p
    I = np.eye(3, dtype=LD)
    for sl in _blocks(len(r_trg), len(r_src)):
        d, r2 = _pairs(r_src, r_trg, sl)
        z = r2 == 0
        y = np.where(z, LD(0), 1 / np.sqrt(np.where(z, LD(1), r2)))
        y3, y5 = y ** 3, y ** 5
        fr = np.einsum("tsk,sk->ts", d, f)
        g = (I[None, None] * (fr * y3)[..., None, None] - f[None, :, :, None] * d[..., None, :] * y3[..., None, None]
             + d[..., :, None] * f[None, :, None, :] * y3[..., None, None]
             - 3 * d[..., :, None] * d[..., None, :] * (fr * y5)[..., None, None])
        G[sl] = g.sum(axis=1) / (8 * PI * eta)
        p[sl] = (fr * y3).sum(axis=1) / (4 * PI)
    return G, p


def stresslet(r_src, S9, r_trg, eta):
    """(G, p) of stresslets S (9 per source, row-major, as the library's f_dl) at r_src"""
    r_src, S, r_trg = _ld(r_src, 3), _ld(S9, 9).reshape(-1, 3, 3), _ld(r_trg, 3)
    eta = LD(eta)
    G, p = np.zeros((len(r_trg), 3, 3), dtype=LD), np.zeros(len(r_trg), dtype=LD)
    if len(r_src) == 0:
        return G, p
    kappa = -3 / (8 * PI * eta)
    I = np.eye(3, dtype=LD)
    Ssym2 = S + np.transpose(S, (0, 2, 1))
    tr = np.trace(S, axis1=1, axis2=2)
    for sl in _blocks(len(r_trg), len(r_src)):
        d, r2 = _pairs(r_src, r_trg, sl)
        z = r2 == 0
        y = np.where(z, LD(0), 1 / np.sqrt(np.where(z, LD(1), r2)))
        y2, y3, y5 = y * y, y ** 3, y ** 5
        A = np.einsum("tsa,sab,tsb->ts", d, S, d)
        h = np.einsum("sab,tsb->tsa", Ssym2, d)
        g = (I[None, None] * A[..., None, None] + d[..., :, None] * h[..., None, :]
             - 5 * d[..., :, None] * d[..., None, :] * (A * y2)[..., None, None]) * y5[..., None, None]
        G[sl] = kappa * g.sum(axis=1)
        p[sl] = 2 * kappa * eta * (A * y5 - tr[None, :] * y3 / 3).sum(axis=1)
    return G, p


def _reg_dist(r2, regularised):
    return np.where(regularised, np.sqrt(r2 + LD(REG) ** 2), np.sqrt(r2))


def rotlet(r_src, L, r_trg, eta):
    """G of rotlet_add_kernel's regularised rotlets (torques L at r_src); no pressure"""
    r_src, L, r_trg = _ld(r_src, 3), _ld(L, 3), _ld(r_trg, 3)
    G = np.zeros((len(r_trg), 3, 3), dtype=LD)
    if len(r_src) == 0:
        return G
    eps3 = np.zeros((3, 3, 3), dtype=LD)
    for i, a, j in ((0, 1, 2), (1, 2, 0), (2, 0, 1)):
        eps3[i, a, j], eps3[i, j, a] = 1, -1
    E = np.einsum("iaj,sa->sij", eps3, L)  # eps_iaj L_a
    for sl in _blocks(len(r_trg), len(r_src)):
        d, r2 = _pairs(r_src, r_trg, sl)
        z = r2 == 0
        D = _reg_dist(r2, r2 < LD(EPS) ** 2)
        D = np.where(z, LD(1), D)
        m = np.cross(L[None, :, :], d)
        g = E[None] / D[..., None, None] ** 3 - 3 * m[..., :, None] * d[..., None, :] / D[..., None, None] ** 5
        G[sl] = np.where(z[..., None, None], LD(0), g).sum(axis=1) / (8 * PI * LD(eta))
    return G


def oseen(r_src, f, r_trg, eta):
    """(G, p) of oseen_contract_add_kernel's regularised point forces f at r_src"""
    r_src, f, r_trg = _ld(r_src, 3), _ld(f, 3), _ld(r_trg, 3)
    G, p = np.zeros((len(r_trg), 3, 3), dtype=LD), np.zeros(len(r_trg), dtype=LD)
    if len(r_src) == 0:
        return G, p
    I = np.eye(3, dtype=LD)
    for sl in _blocks(len(r_trg), len(r_src)):
        d, r2 = _pairs(r_src, r_trg, sl)
        z = r2 == 0
        D = _reg_dist(r2, np.sqrt(r2) <= LD(EPS))
        D = np.where(z, LD(1), D)
        fr = np.einsum("tsk,sk->ts", d, f)
        y3, y5 = D ** -3, D ** -5
        g = (I[None, None] * (fr * y3)[..., None, None] - f[None, :, :, None] * d[..., None, :] * y3[..., None, None]
             + d[..., :, None] * f[None, :, None, :] * y3[..., None, None]
             - 3 * d[..., :, None] * d[..., None, :] * (fr * y5)[..., None, None])
        G[sl] = np.where(z[..., None, None], LD(0), g).sum(axis=1) / (8 * PI * LD(eta))
        p[sl] = np.where(z, LD(0), fr * y3).sum(axis=1) / (4 * PI)
    return G, p


def background(n_trg, comp, scale):
    G = np.zeros((n_trg, 3, 3), dtype=LD)
    for j in range(3):
        G[:, j, comp[j]] += LD(scale[j])
    return G


def double_layer(normals, density, eta):
    """f_dl = 2 eta n (x) rho, 9 per node"""
    n, rho = _ld(normals, 3), _ld(density, 3)
    return (2 * LD(eta) * n[:, :, None] * rho[:, None, :]).reshape(-1, 9)


def trapezoid_weights(n_nodes, length):
    w = np.full(n_nodes, LD(2))
    w[0] = w[-1] = 1
    return LD(0.5) * LD(length) * (w / LD(n_nodes - 1))


def rigid_gradient(omega):
    w0, w1, w2 = omega
    return np.array([[0, -w2, w1], [w2, 0, -w0], [-w1, w0, 0]], dtype=LD)


def frame_gradient(fib, shell, body, pts, pf, ptq, bg, eta, r, inside=None, uw=None):
    """The whole frame: fibers (trapezoid-weighted Stokeslets, no self subtraction), body surfaces (stresslets) and
    centres (Stokeslets of the forces, rotlets of the torques), periphery (stresslets), point sources (Oseen + rotlet),
    background (comp, scale, uniform).  inside: per body, the targets its interior test takes (the last wins), with
    uw[b] = [U, omega]: there G is the rigid gradient and p NaN.  Returns (G, p) in long double."""
    r = _ld(r, 3)
    G, p = np.zeros((len(r), 3, 3), dtype=LD), np.zeros(len(r), dtype=LD)

    def add(gp):
        G[...] += gp[0]
        p[...] += gp[1]

    if len(fib["n_nodes"]):
        w = np.concatenate([trapezoid_weights(n, L) for n, L in zip(fib["n_nodes"], fib["lengths"])])
        add(stokeslet(fib["pos"], _ld(fib["forces"], 3) * w[:, None], r, eta))
    if len(body["centers"]):
        add(stresslet(body["pos"], double_layer(body["normals"], body["density"], eta), r, eta))
        add(stokeslet(body["centers"], body["forces"], r, eta))
        G[...] += rotlet(body["centers"], body["torques"], r, eta)
    if len(shell["pos"]):
        add(stresslet(shell["pos"], double_layer(shell["normals"], shell["density"], eta), r, eta))
    if len(pts):
        add(oseen(pts, pf, r, eta))
        G[...] += rotlet(pts, ptq, r, eta)
    if bg is not None:
        G[...] += background(len(r), bg[0], bg[1])
    for b, m in enumerate(inside or []):
        G[m] = rigid_gradient(_ld(uw[b][3:], 1).reshape(-1))
        p[m] = np.nan
    return G, p

"""Extended-precision restatement of the body block and the fiber-body links (body_ops.cuh, skb_body.cu) -- TEST
INFRASTRUCTURE ONLY.  Same dict conventions as tests/system_reference.py.

Every function takes float64 inputs and evaluates in `dtype`: np.longdouble gives `ext`, the exactly rounded function
of those inputs up to 2^-64; np.float64 gives a float64 restatement.  absolute=True gives the error scale S: every
input by its absolute value and every subtraction an addition, except that a difference of two float64 inputs (a node
minus a centre, a nucleation site minus a centre) enters as |a - b|, because one rounded subtraction errs by u relative
to its result.  Sums run in the kernels' order (strided lanes, then their fixed reduction tree), so the float64
restatement rounds like the kernels up to FMA contraction.

A device value passes when |dev - ext| <= K u S entry by entry, u = 2^-53.  Each K below is the count of roundings on
the longest path from the float64 inputs to the entry (first-order: an FMA counts one, a product or quotient one, a
sum of k terms k - 1 along its deepest operand), plus SLACK:

    K_LINK_ROWS        the seven link conditions: s = site - c (1), w x s (2), -U - w x s (1) = 4; the tension row
                       xs.U (3), xs x s (1 + 2), its dot with w (3), the difference (1) = 10; the rotational row |s|^2
                       (1 + 3), sqrt (1), 1/ (1), s / |s| (1), (s/|s|) x w (2) = 9.  Base 10.
    k_ft(n, m)         a body's force and torque: xss / xsss as a lane sum of ceil(n/32) FMAs and a 5-level shuffle
                       tree, times (2/L)^2 or ^3 (3 + 1); the torque's crosses and its three-term sum (s 1, cross 2,
                       x E 1, sums 2) = ceil(n/32) + 5 + 4 + 6 = ceil(n/32) + 15; then body_sum_kernel adds the m bound
                       fibers one after the other, m - 1 more.  n is the largest node count among them.
    k_flow(n_src)      the centre Stokeslet and rotlet at one target: per source d (1), |d|^2 (3), 1/|d| by
                       MUFU + Newton (3), f.d (3), (f.d)/|d|^2 (3), d q + f (1), y v (1): 15 along the deepest path,
                       counted generously as 20; n_src - 1 for the sum over the centres; 1/eta, /(8 pi) and the scaling
                       multiply, 3; the rotlet's own path (|d|^3 and its reciprocal, the cross) is shorter.
                       Base n_src + 23.  The body node rows (and a fiber's node 0) see F and L with their own error:
                       K = k_flow(n_src) + k_ft of the worst body, with S built from S_F and S_L.
    K_NODE             a body node row of body_matvec_kernel: d / w (1), times e and three-term sum (3), x - c (1),
                       w x (x - c) (2), U + that (1), the two outer sums (2) = 9 ... counted as 10.
    k_kt(n)            the six rows -K^T lambda + U: ceil(n/256) strided terms per thread, an 8-level tree over the
                       256 threads, the final difference (1), and for the torque rows x - c (1) and the cross (2):
                       ceil(n/256) + 12.
    k_gemv(m)          a row of the body preconditioner (fiber_gemv_kernel<0>): ceil(m/8) FMAs per column slice, then
                       the 8 slice partials added one after the other (7): ceil(m/8) + 7.
"""
import numpy as np

U = 2.0 ** -53
SLACK = 4
K_LINK_ROWS = 10 + SLACK
K_NODE = 10 + SLACK

# planted defects a criterion must catch.  Links: the sign of omega x s in v_fiber; length_prev_ in place of length_ in
# xsss or in xss; the last bound fiber of a body dropped from its sum.  Body rows: the sign of omega x (x_i - c); d w in
# place of d / w; the torque sum as lambda x (x_i - c); a K^T lambda reduction that skips node 256.  Preconditioner: the
# second 32-row block of a body answered with the third block's rows.
LINK_DEFECTS = ("omega_site_sign", "xsss_length_prev", "xss_length_prev", "drop_last_fiber")
BODY_DEFECTS = ("node_omega_sign", "d_times_w", "torque_reversed", "skip_node_256")
GEMV_DEFECTS = ("shift_block_32",)


def k_ft(n_max, n_bound):
    return int(np.ceil(n_max / 32)) + 15 + max(n_bound - 1, 0) + SLACK


def k_flow(n_src):
    return n_src + 23 + SLACK


def k_kt(n):
    return int(np.ceil(n / 256)) + 12 + SLACK


def k_gemv(m):
    return int(np.ceil(m / 8)) + 7 + SLACK


def ratio(got, ext, S):
    """|got - ext| / (u S) entry by entry (float64); a structural zero (S = 0) counts 0 if exact, inf if not"""
    d = np.abs(np.asarray(got, dtype=np.float64).astype(np.longdouble) - ext).astype(np.float64)
    S = np.asarray(S, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(S > 0, d / (U * S), np.where(d == 0, 0.0, np.inf))


class _Ar:
    """the arithmetic of one evaluation: dtype, and the sign a subtraction takes (+1 for S)"""

    def __init__(self, dtype, absolute):
        self.f, self.absolute = dtype, absolute
        self.sg = 1.0 if absolute else -1.0

    def v(self, a):                       # a float64 input
        a = np.asarray(a, dtype=np.float64).astype(self.f)
        return np.abs(a) if self.absolute else a

    def diff(self, a, b):                 # a difference of two float64 inputs
        d = np.asarray(a, dtype=np.float64).astype(self.f) - np.asarray(b, dtype=np.float64).astype(self.f)
        return np.abs(d) if self.absolute else d

    def cross(self, a, b):
        s = self.sg
        return np.stack([a[..., 1] * b[..., 2] + s * (a[..., 2] * b[..., 1]),
                         a[..., 2] * b[..., 0] + s * (a[..., 0] * b[..., 2]),
                         a[..., 0] * b[..., 1] + s * (a[..., 1] * b[..., 0])], axis=-1)


def lane_sum(t, lanes, tree=True):
    """sum over axis 0 as a kernel does it: lane l adds items l, l + lanes, ... in turn, then the lanes are combined by a
    halving tree (the shuffle tree of fiber_link_kernel, the shared-memory tree of body_matvec_kernel) or, tree=False,
    one after the other (the slice partials of fiber_gemv_kernel)"""
    t = np.asarray(t)
    n = t.shape[0]
    rows = max(1, -(-n // lanes))
    p = np.zeros((rows * lanes,) + t.shape[1:], dtype=t.dtype)
    p[:n] = t
    p = p.reshape((rows, lanes) + t.shape[1:])
    acc = p[0].copy()
    for k in range(1, rows):
        acc = acc + p[k]
    if tree:
        while acc.shape[0] > 1:
            h = acc.shape[0] // 2
            acc = acc[:h] + acc[h:]
        return acc[0]
    s = acc[0]
    for k in range(1, lanes):
        s = s + acc[k]
    return s


def link_terms(fib, ops, links, bodies, x_fibers, x_bodies, dtype=np.longdouble, absolute=False, defect=None):
    """fiber_link_kernel + body_sum_kernel (calculate_link_conditions, the implemented reading): returns (link
    (n_fibers, 7), contrib (n_fibers, 6) = [F | L] per bound fiber, ft (n_bodies, 6) = the bodies' sums in container
    order).  Free fibers: zeros."""
    assert defect is None or defect in LINK_DEFECTS, defect
    a = _Ar(dtype, absolute)
    f, sg = a.f, a.sg
    ng = sg                                # a negation (dropped in S)
    n_nodes = [int(n) for n in fib["n_nodes"]]
    nfib, nb = len(n_nodes), len(bodies["n_nodes"])
    sol_off = np.concatenate([[0], np.cumsum(3 * np.asarray(bodies["n_nodes"], dtype=np.int64) + 6)])
    fib_off = np.concatenate([[0], np.cumsum(n_nodes)]).astype(int)
    link = np.zeros((nfib, 7), dtype=f)
    contrib = np.zeros((nfib, 6), dtype=f)
    for i, n in enumerate(n_nodes):
        b = int(links["body"][i])
        if b < 0:
            continue
        s = a.diff(links["site"][i], bodies["centers"][b])
        o = 4 * fib_off[i]
        x = a.v(x_fibers[o:o + 3 * n]).reshape(3, n)
        T0 = a.v(x_fibers[o + 3 * n])
        xs0 = a.v(ops["xs"][fib_off[i]])
        L = f(fib["lengths"][i])
        Lp = f(ops["length_prev"][i])
        D2, D3 = a.v(np.asarray(ops["D_2_0"][n])[:, 0]), a.v(np.asarray(ops["D_3_0"][n])[:, 0])
        a2 = lane_sum((x * D2).T, 32)
        a3 = lane_sum((x * D3).T, 32)
        q2 = (f(2.0) / (Lp if defect == "xss_length_prev" else L)) ** 2
        q3 = (f(2.0) / (Lp if defect == "xsss_length_prev" else L)) ** 3
        xss, xsss = q2 * a2, q3 * a3
        E = a.v(links["rigidity"][i])
        contrib[i, :3] = ng * E * xsss + xs0 * T0
        contrib[i, 3:] = ng * E * a.cross(s, xsss) + a.cross(s, xs0) * T0 + E * a.cross(xs0, xss)
        j = int(sol_off[b]) + 3 * int(bodies["n_nodes"][b])
        Ub, w = a.v(x_bodies[j:j + 3]), a.v(x_bodies[j + 3:j + 6])
        ws = a.cross(w, s)
        link[i, :3] = ng * Ub + (-ng if defect == "omega_site_sign" else ng) * ws
        link[i, 3] = ng * np.sum(xs0 * Ub) + np.sum(a.cross(xs0, s) * w)
        sn = s / np.sqrt(np.sum(s * s))
        link[i, 4:] = a.cross(sn, w)
    ft = np.zeros((nb, 6), dtype=f)
    for b in range(nb):
        mine = [i for i in range(nfib) if int(links["body"][i]) == b]
        if defect == "drop_last_fiber" and mine:
            mine = mine[:-1]
        for i in mine:
            ft[b] = ft[b] + contrib[i]
    return link, contrib, ft


def centre_flow(r_trg, centers, F, L, eta, dtype=np.longdouble, absolute=False):
    """the centre part of BodyContainer::flow at the targets (skb_matvec.cu bodies_dev): the Stokeslet of the bodies'
    forces F through the plain pair kernel, the rotlet of their torques L (rotlet_add_kernel).  F and L are taken as
    given in `dtype` (ext F / L, or S_F / S_L with absolute=True); the targets stay clear of the centres' regularisation."""
    a = _Ar(dtype, absolute)
    f = a.f
    F, L = np.asarray(F, dtype=f), np.asarray(L, dtype=f)
    d = a.diff(np.asarray(r_trg)[:, None, :], np.asarray(centers)[None, :, :])     # (n_trg, n_src, 3)
    y = 1 / np.sqrt(np.sum(d * d, axis=2))                                           # 1/|d|
    fd = np.sum(F[None] * d, axis=2)
    v = F[None] + d * (fd * y * y)[..., None]
    pi = f(np.pi)
    stok = np.sum(y[..., None] * v, axis=1) * ((f(1) / f(eta)) / (f(8) * pi))
    rot = np.sum((y ** 3)[..., None] * a.cross(L[None], d), axis=1) * (f(1) / (f(8) * pi * f(eta)))
    return stok + rot


def body_rows(bodies, v_bodies, x_bodies, dtype=np.longdouble, absolute=False, defect=None):
    """body_matvec_kernel (SphericalBody::matvec per body) in the x_bodies layout: node rows -(cx + cy + cz) - (U + w x
    (x_i - c)) + v, then the six rows -K^T lambda + U."""
    assert defect is None or defect in BODY_DEFECTS, defect
    a = _Ar(dtype, absolute)
    f, sg = a.f, a.sg
    ng = sg                                # a negation (dropped in S)
    n_nodes = [int(n) for n in bodies["n_nodes"]]
    node_off = np.concatenate([[0], np.cumsum(n_nodes)]).astype(int)
    sol_off = np.concatenate([[0], np.cumsum(3 * np.asarray(n_nodes, dtype=np.int64) + 6)]).astype(int)
    res = np.empty(int(sol_off[-1]), dtype=f)
    for b, n in enumerate(n_nodes):
        p, s = node_off[b], sol_off[b]
        d = a.v(x_bodies[s:s + 3 * n]).reshape(n, 3)
        Ub, om = a.v(x_bodies[s + 3 * n:s + 3 * n + 3]), a.v(x_bodies[s + 3 * n + 3:s + 3 * n + 6])
        w = a.v(bodies["weights"][p:p + n])[:, None]
        dw = d * w if defect == "d_times_w" else d / w
        c = dw[:, 0:1] * a.v(bodies["ex"][p:p + n]) + dw[:, 1:2] * a.v(bodies["ey"][p:p + n]) + \
            dw[:, 2:3] * a.v(bodies["ez"][p:p + n])
        rr = a.diff(bodies["pos"][p:p + n], bodies["centers"][b])
        om_r = a.cross(om, rr) if defect != "node_omega_sign" else a.cross(rr, om)
        v = a.v(v_bodies[p:p + n])
        res[s:s + 3 * n] = (ng * c + ng * (Ub + om_r) + v).reshape(-1)
        r_d = a.cross(d, rr) if defect == "torque_reversed" else a.cross(rr, d)
        terms = np.concatenate([d, r_d], axis=1)
        if defect == "skip_node_256" and n > 256:
            terms[256] = 0
        res[s + 3 * n:s + 3 * n + 6] = ng * lane_sum(terms, 256) + np.concatenate([Ub, om])
    return res


def gemv_rows(A, x, rows=None, dtype=np.longdouble, absolute=False, defect=None):
    """(A x)[rows] as fiber_gemv_kernel<0> sums it (column slices j = q mod 8, then the slices in turn); rows None: all.
    shift_block_32: rows 32 .. 63 take the values of rows 64 .. 95."""
    assert defect is None or defect in GEMV_DEFECTS, defect
    a = _Ar(dtype, absolute)
    m = A.shape[1]
    rows = np.arange(A.shape[0]) if rows is None else np.asarray(rows)
    src = rows.copy()
    if defect == "shift_block_32":
        src = np.where((rows >= 32) & (rows < 64) & (rows + 32 < A.shape[0]), rows + 32, rows)
    M = a.v(A[src])                       # (len(rows), m)
    xv = a.v(x)
    return lane_sum((M * xv[None, :]).T, 8, tree=False)


def ext_and_scale(fn, *args, **kw):
    """(ext, S) of one of the functions above"""
    return fn(*args, dtype=np.longdouble, **kw), fn(*args, dtype=np.longdouble, absolute=True, **kw)

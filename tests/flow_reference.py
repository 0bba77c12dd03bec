"""Extended-precision restatement of the flows at targets and of the hydrodynamic velocity v_all of skb_flow_matvec
(skb_matvec.cu: fibers_dev, bodies_dev, periphery_dev, add_sources, velocity_dev, matvec_core; aux_kernels.cuh:
fiber_self_subtract_kernel, oseen_contract_add_kernel, rotlet_add_kernel, background_add_kernel) and of the listener's
velocity_field (listener_kernels.cuh interior_replace_kernel) -- TEST INFRASTRUCTURE ONLY.  Conventions of
tests/pair_sum_reference.py and tests/body_block_reference.py (U, ratio): every function takes float64 inputs and
returns, per target row, (ext, S, K):

    ext  in np.longdouble, the function of the float64 inputs the kernels compute, with the kernels' own branch rules;
    S    the same sum with every term by its absolute value (|d| for a rounded difference of coordinates, |f| . |d| for a
         dot product, |a b| + |c d| for a cross-product component);
    K    (per row) the worst-case rounding count of the device's evaluation, fixed from the kernel source below.

A device row passes when |dev - ext| <= K u S component by component, u = 2^-53.

The pair sums (the fibers' Stokeslets, the periphery's and the bodies' stresslets, the bodies' centre Stokeslets) are
pair_sum_reference.pair_rows, with the packed strengths restated bit for bit in float64 (trapezoid_weights,
weighted_forces, double_layer_sym6) and their K from that module: k_plain_bound, k_cross, and the symmetric kernel's
k_sym_rows, which a caller passes in where the symmetric path can run (it needs the launch plan).

Branch rules.  Every decision is made on the float64 value the kernel forms, never on the exact one.  The kernels' r^2 is
dx*dx + dy*dy + dz*dz, which nvcc may contract into FMAs; each decision is taken on both forms and a geometry on which
they disagree is refused (ValueError), so a test cannot depend on the contraction.  Axis-aligned pairs (dy = dz = 0)
make every form exact.
    fiber self term      d = src - trg; a pair is skipped when the float64 r^2 == 0 and regularised when the float64
                         r = sqrt(r^2) <= EPS: G = c (f / D + d (d . f) / D^3), D = r or sqrt(r^2 + REG2)
                         (kernels.cpp:146-195, applied by fcfd.cpp:203-210).  The pair kernels mask r^2 < DBL_MIN;
                         the self term skips r^2 == 0 only.  So a pair of one fiber's nodes whose float64 r^2 is
                         subnormal is not in the pair sum but is subtracted, regularised -- the rule pinned here, and
                         one more instance of the by-design non-cancellation within EPS: there the pair sum holds the
                         unregularised pair and the self term removes the regularised one.
    point sources        oseen_contract_add_kernel: the self term's rule (r == 0 skipped, r <= EPS regularised);
                         rotlet_add_kernel: d = trg - src, D = sqrt(REG2 + r^2) when r^2 < EPS2, else r; no r == 0
                         skip (a coincident pair has L x d = 0 and adds exactly 0).  The bodies' centre rotlets are the
                         same kernel.
    background           u_j += uniform_j + r[c_j] scale_j.
    interior             (velocity_field) bodies in order, the last whose float64 interior test holds wins; its rows
                         are U + omega x (x - c), bitwise, every operation rounded on its own.

K (first-order counts in u; an FMA counts one; relative to the pair's absolute term):
    c = 1 / (8 pi eta): M_PI rounded, * eta, 1 /                                                         3
    K_OSEEN_PAIR -- fiber_self_subtract_kernel and oseen_contract_add_kernel, per pair:
        d_k = src - trg 1;  r^2: d rounded (2), three products / sums (3) 5;  r = sqrt(r^2): 2.5 + 1 = 3.5
        unregularised:  fr = c / r: 3 + 3.5 + 1 = 7.5;  gr = c / (r r r): 3 + (3 x 3.5 + 2) + 1 = 16.5
        regularised:    r r + REG2: 7 + 1 + 1 = 9;  sqrt 4.5 + 1;  1 / 1: 6.5;  fr = c di 10.5;  gr = c di di di 25.5
        d . f: d rounded, product, two sums 4;  dot = gr (d . f): 25.5 + 4 + 1 = 30.5
        d_k dot: 1 + 30.5 + 1 = 32.5;  fr f_k: 11.5;  their sum 33.5                                       34
    K_ROTLET_PAIR -- rotlet_add_kernel, per pair, its post-scale included:
        d 1;  r^2 5;  D: sqrt(r^2) 3.5 or sqrt(REG2 + r^2) 4;  1 / (D D D): 3 x 4 + 2 + 1 = 15
        L x d component: d rounded, product, difference 3;  fr (L x d): 15 + 3 + 1 = 19;  c a: 3 + 1 = 4    23
    k_self(n)   = K_OSEEN_PAIR + n (the sequential j sum) + 1 (the subtraction from the row)
    k_points(m) = K_OSEEN_PAIR + m (the sum over the point sources)
    k_rotlet(m) = K_ROTLET_PAIR + m (the sum over the sources)
    K_BG        = 2 (the product r[c_j] scale_j and the sum with uniform_j)
    each of these + K_REF(N) (pair_sum_reference.k_ref of the N terms summed in long double) + SLACK (4).
    compose() -- a row made of parts: K_row = max over the parts of K_part + one rounding per part for the accumulate
    that brings it into the row (the pair kernels' accumulate, add_inplace_kernel, the += / -= of the small kernels, the
    1/eta folded into a post-scale), and S_row the sum of the parts' S.  Each part errs by at most K_part u S_part and
    every accumulate by u times a partial sum bounded by S_row, so the row errs by at most K_row u S_row.

Planted defects (defect=), each a slip the kernels or their composition could make; tests/test_flow_ext_cpu.py shows
that each misses its bound by orders of magnitude on some row:
    self_j_short         the self term's j loop stops at n - 1
    self_no_reg          the self term's regularised branch dropped (unregularised at every r > 0)
    self_eps_strict      the self term regularises at r < EPS instead of r <= EPS
    self_window_offset   the self term writes window rows at off + i instead of off + i - node_begin
    weights_not_halved   the trapezoid weights not halved at the fiber ends
    rotlet_eps_le        the rotlet regularises at r^2 <= EPS2
    point_r0_kept        a point source at r == 0 is not skipped
    bg_component         the background takes r[:, j] instead of r[:, c_j]
    periphery_no_eta     the periphery's post-scale without its 1/eta
    interior_first_wins  the interior test lets the first matching body win
    self_twice           the self term subtracted twice (the grouped path: after the pull and before it)
    self_skipped         the self term not subtracted (the grouped path)
"""
import numpy as np

import pair_sum_reference as ps
from body_block_reference import U, ratio  # noqa: F401  (for the tests)

LD = np.longdouble
EPS = 1e-5                               # kEps (skb_matvec.cu; include/kernels.hpp:38-46)
REG = 5e-3                               # kReg
REG2 = np.float64(REG) * np.float64(REG)  # kReg * kReg and kEps * kEps, formed in float64 as the host passes them
EPS2 = np.float64(EPS) * np.float64(EPS)
SLACK = 4
K_OSEEN_PAIR = 34
K_ROTLET_PAIR = 23
K_BG = 2

DEFECTS = ("self_j_short", "self_no_reg", "self_eps_strict", "self_window_offset", "weights_not_halved",
           "rotlet_eps_le", "point_r0_kept", "bg_component", "periphery_no_eta", "interior_first_wins", "self_twice",
           "self_skipped")


def k_self(n):
    return K_OSEEN_PAIR + n + 1 + ps.k_ref(n) + SLACK


def k_points(m):
    return K_OSEEN_PAIR + m + ps.k_ref(m) + SLACK


def k_rotlet(m):
    return K_ROTLET_PAIR + m + ps.k_ref(m) + SLACK


def c_of(eta):
    """the exact 1 / (8 pi eta)"""
    return LD(1) / (LD(8) * ps.PI * LD(eta))


# ---- parts and rows -----------------------------------------------------------------------------------------------
def part(ext, S, K):
    ext, S = np.asarray(ext, dtype=LD), np.asarray(S, dtype=LD)
    return ext, S, np.broadcast_to(np.asarray(K, dtype=np.float64), ext.shape[:1]).copy()


def compose(*parts):
    """(ext, S, K) of a row made of parts, each brought into the row by one accumulate"""
    parts = [p for p in parts if p is not None]
    ext = sum(p[0] for p in parts)
    S = sum(p[1] for p in parts)
    K = np.max(np.stack([p[2] for p in parts]), axis=0) + len(parts)
    return ext, S, K


def neg(p):
    return -p[0], p[1], p[2]


def take(p, rows):
    return p[0][rows], p[1][rows], p[2][rows]


def concat(*ps_):
    return tuple(np.concatenate([p[k] for p in ps_]) for k in range(3))


# ---- branch decisions on the kernels' float64 r^2 ---------------------------------------------------------------------
def _decide(d64, rule):
    """rule(r2) -> tuple of bool arrays, taken on the plain float64 r^2 and on its contracted form; refused where they
    differ"""
    plain = d64[..., 0] * d64[..., 0] + d64[..., 1] * d64[..., 1] + d64[..., 2] * d64[..., 2]
    a = rule(plain)
    b = rule(ps.r2_kernel(d64[..., 0], d64[..., 1], d64[..., 2]))
    for x, y in zip(a, b):
        if not np.array_equal(x, y):
            raise ValueError("a branch of the flow kernels depends on FMA contraction at this geometry")
    return a


def _oseen_terms(t, s, f, eta, skip_rule, reg_rule):
    """(term, aterm) (R, n, 3) of G(s - t) f, the regularised Oseen tensor of oseen_contract_add_kernel /
    fiber_self_subtract_kernel, scale c included"""
    d64 = s[None, :, :] - t[:, None, :]

    def rule(r2):
        r = np.sqrt(r2)
        return skip_rule(r2), reg_rule(r)
    skip, reg = _decide(d64, rule)
    d = s.astype(LD)[None, :, :] - t.astype(LD)[:, None, :]
    r2 = (d * d).sum(axis=-1)
    y = 1 / np.sqrt(np.where(reg, r2 + LD(REG2), np.where(skip, LD(1), r2)))
    y = np.where(skip, LD(0), y) * c_of(eta)
    y3 = np.where(skip, LD(0), (y / c_of(eta)) ** 3 * c_of(eta))
    F = f.astype(LD)[None, :, :]
    A, ad = np.abs(F), np.abs(d)
    term = y[..., None] * F + d * (y3 * (d * F).sum(axis=-1))[..., None]
    aterm = y[..., None] * A + ad * (y3 * (ad * A).sum(axis=-1))[..., None]
    return term, aterm


def _skip_r0(r2):
    return r2 == 0.0


def _reg_le(r):
    return r <= EPS


# ---- the small kernels --------------------------------------------------------------------------------------------
def point_oseen(r_trg, pts, forces, eta, defect=None):
    """oseen_contract_add_kernel at every target: (ext, S, K)"""
    t, s = np.asarray(r_trg, dtype=np.float64), np.asarray(pts, dtype=np.float64)
    skip = (lambda r2: np.zeros(r2.shape, dtype=bool)) if defect == "point_r0_kept" else _skip_r0
    term, aterm = _oseen_terms(t, s, np.asarray(forces, dtype=np.float64), eta, skip, _reg_le)
    return part(term.sum(axis=1), aterm.sum(axis=1), k_points(s.shape[0]))


def rotlet(r_trg, src, torques, eta, defect=None):
    """rotlet_add_kernel at every target: (ext, S, K)"""
    t, s = np.asarray(r_trg, dtype=np.float64), np.asarray(src, dtype=np.float64)
    d64 = t[:, None, :] - s[None, :, :]
    reg, = _decide(d64, lambda r2: ((r2 <= EPS2) if defect == "rotlet_eps_le" else (r2 < EPS2),))
    d = t.astype(LD)[:, None, :] - s.astype(LD)[None, :, :]
    r2 = (d * d).sum(axis=-1)
    D = np.sqrt(np.where(reg, r2 + LD(REG2), r2))
    y3 = np.where(D > 0, 1 / np.where(D > 0, D, LD(1)) ** 3, LD(0))
    L = np.asarray(torques, dtype=np.float64).astype(LD)[None]
    cr = np.stack([L[..., 1] * d[..., 2] - L[..., 2] * d[..., 1], L[..., 2] * d[..., 0] - L[..., 0] * d[..., 2],
                   L[..., 0] * d[..., 1] - L[..., 1] * d[..., 0]], axis=-1)
    A, ad = np.abs(L), np.abs(d)
    acr = np.stack([A[..., 1] * ad[..., 2] + A[..., 2] * ad[..., 1], A[..., 2] * ad[..., 0] + A[..., 0] * ad[..., 2],
                    A[..., 0] * ad[..., 1] + A[..., 1] * ad[..., 0]], axis=-1)
    c = c_of(eta)
    return part(c * (y3[..., None] * cr).sum(axis=1), c * (y3[..., None] * acr).sum(axis=1), k_rotlet(s.shape[0]))


def background(r_trg, comp, scale, uniform, defect=None):
    """background_add_kernel: (ext, S, K)"""
    t = np.asarray(r_trg, dtype=np.float64).astype(LD)
    comp = [0, 1, 2] if defect == "bg_component" else [int(c) for c in comp]
    sc, un = np.asarray(scale, dtype=np.float64).astype(LD), np.asarray(uniform, dtype=np.float64).astype(LD)
    return part(un[None] + t[:, comp] * sc[None], np.abs(un)[None] + np.abs(t[:, comp]) * np.abs(sc)[None],
                K_BG + SLACK)


def self_term(r_fib, n_nodes, wf, eta, nodes, defect=None):
    """fiber_self_subtract_kernel's contribution, -sum_j G(x_j - x_i) wf_j, at rows whose fiber node is nodes[row]
    (-1: a row without a self term, exactly 0)"""
    r_fib, wf = np.asarray(r_fib, dtype=np.float64), np.asarray(wf, dtype=np.float64)
    nodes = np.asarray(nodes, dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(n_nodes)]).astype(np.int64)
    ext = np.zeros((nodes.size, 3), dtype=LD)
    S = np.zeros((nodes.size, 3), dtype=LD)
    K = np.zeros(nodes.size)
    fiber = np.searchsorted(off, nodes, side="right") - 1
    reg = {"self_no_reg": lambda r: np.zeros(r.shape, dtype=bool),
           "self_eps_strict": lambda r: r < EPS}.get(defect, _reg_le)
    for fi in np.unique(fiber[nodes >= 0]):
        rows = np.flatnonzero((fiber == fi) & (nodes >= 0))
        a, n = off[fi], int(n_nodes[fi])
        m = n - 1 if defect == "self_j_short" else n
        for c0 in range(0, rows.size, max(1, (1 << 19) // n)):
            rr = rows[c0:c0 + max(1, (1 << 19) // n)]
            term, aterm = _oseen_terms(r_fib[nodes[rr]], r_fib[a:a + m], wf[a:a + m], eta, _skip_r0, reg)
            ext[rr], S[rr] = -term.sum(axis=1), aterm.sum(axis=1)
        K[rows] = k_self(n)
    return ext, S, K


# ---- the flows of the classes -------------------------------------------------------------------------------------
def fiber_weights(fib, defect=None):
    n_nodes, lengths = fib["n_nodes"], fib["lengths"]
    if defect == "weights_not_halved":
        return np.concatenate([0.5 * np.float64(L) * (np.full(n, 2.0) / np.float64(n - 1))
                               for n, L in zip(n_nodes, lengths)])
    return ps.trapezoid_weights(n_nodes, lengths)


def fiber_pairs(fib, r_trg, eta, k=None, defect=None):
    """the Stokeslet sum of the fibers' weighted forces at r_trg (fibers_dev's pair sum): (ext, S, K); K default the
    plain and cross kernels' bound, k (scalar or per row) raises it (the symmetric kernel's k_sym_rows)"""
    n = fib["pos"].shape[0]
    wf = ps.weighted_forces(fib["forces"], fiber_weights(fib, defect))
    e, S = ps.pair_rows("sl", fib["pos"], wf, r_trg, scale=ps.scale_of("sl", eta))
    K = max(ps.k_plain_bound("sl", n), ps.k_cross("sl", n))
    return part(e, S, np.maximum(K, 0 if k is None else k))


def fiber_flow(fib, r_trg, eta, subtract_self=False, k=None, nodes=None, defect=None):
    """Flow.fiber_flow: the pair sum and, with subtract_self, the self term at the leading rows (the fiber nodes) or at
    rows whose fiber node is nodes[row]"""
    p = fiber_pairs(fib, r_trg, eta, k, defect)
    if not subtract_self:
        return compose(p)
    n = fib["pos"].shape[0]
    if nodes is None:
        nodes = np.where(np.arange(len(r_trg)) < n, np.arange(len(r_trg)), -1)
    wf = ps.weighted_forces(fib["forces"], fiber_weights(fib, defect))
    return compose(p, self_term(fib["pos"], fib["n_nodes"], wf, eta, nodes, defect))


def periphery_flow(shell, r_trg, eta, k=None, defect=None):
    """periphery_dev: the stresslet of 2 eta n (x) rho through its sym6, post-scaled by -3 / (8 pi eta)"""
    n = shell["pos"].shape[0]
    s6 = ps.double_layer_sym6(shell["normals"], shell["density"], eta)
    e, S = ps.pair_rows("dl6", shell["pos"], s6, r_trg,
                        scale=ps.scale_of("dl6", 1.0 if defect == "periphery_no_eta" else eta))
    K = max(ps.k_plain_bound("dl6", n), ps.k_cross("dl6", n))
    return part(e, S, np.maximum(K, 0 if k is None else k))


def body_flow(body, r_trg, eta, defect=None):
    """bodies_dev: the surface stresslet, the centre Stokeslets of the forces and the centre rotlets of the torques;
    the three parts (the caller composes them into its row)"""
    if len(body["centers"]) == 0:
        return []
    s6 = ps.double_layer_sym6(body["normals"], body["density"], eta)
    e, S = ps.pair_rows("dl6", body["pos"], s6, r_trg, scale=ps.scale_of("dl6", eta))
    ec, Sc = ps.pair_rows("sl", body["centers"], body["forces"], r_trg, scale=ps.scale_of("sl", eta))
    return [part(e, S, ps.k_plain_bound("dl6", body["pos"].shape[0])),
            part(ec, Sc, ps.k_plain_bound("sl", len(body["centers"]))),
            rotlet(r_trg, body["centers"], body["torques"], eta, defect)]


def sources(r_trg, eta, points=None, bg=None, defect=None):
    """add_sources: the point sources' Oseen and rotlet parts and the background part"""
    out = []
    if points is not None and len(points[0]):
        pts, pf, ptq = points
        out += [point_oseen(r_trg, pts, pf, eta, defect), rotlet(r_trg, pts, ptq, eta, defect)]
    if bg is not None:
        out.append(background(r_trg, *bg, defect=defect))
    return out


def velocity_at_targets(fib, shell, body, r_trg, eta, points=None, bg=None, k_fib=None, defect=None):
    """velocity_dev: fibers (no self term), bodies, periphery, then the point sources and the background"""
    parts = []
    if fib["pos"].shape[0]:
        parts.append(fiber_pairs(fib, r_trg, eta, k_fib, defect))
    parts += body_flow(body, r_trg, eta, defect)
    if shell["pos"].shape[0]:
        parts.append(periphery_flow(shell, r_trg, eta, defect=defect))
    parts += sources(r_trg, eta, points, bg, defect)
    if not parts:
        z = np.zeros((len(r_trg), 3), dtype=LD)
        return z, z.copy(), np.zeros(len(r_trg))
    return compose(*parts)


def interior(r, body, kind, radii, uw, defect=None):
    """interior_replace_kernel: (mask, rigid) -- the rows some body's interior test takes and there, bitwise, U + omega x
    (x - c) of the last such body (first with interior_first_wins)"""
    r = np.asarray(r, dtype=np.float64)
    mask = np.zeros(len(r), dtype=bool)
    out = np.zeros((len(r), 3))
    order = range(len(body["centers"]))
    if defect == "interior_first_wins":
        order = reversed(order)
    for b in order:
        c, k, rad = np.asarray(body["centers"][b]), int(kind[b]), np.asarray(radii[b], dtype=np.float64)
        if k == 0:
            continue
        d = r - c
        if k == 1:
            m = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]) < rad[0]
        else:
            q = [d[:, j] * d[:, j] / rad[j] / rad[j] for j in range(3)]
            m = (q[0] + q[1]) + q[2] < 1.0
        w = np.asarray(uw[b][3:], dtype=np.float64)
        v = np.asarray(uw[b][:3], dtype=np.float64) + np.stack(
            [w[1] * d[:, 2] - w[2] * d[:, 1], w[2] * d[:, 0] - w[0] * d[:, 2], w[0] * d[:, 1] - w[1] * d[:, 0]], axis=1)
        out[m] = v[m]
        mask |= m
    return mask, out


def velocity_field(fib, shell, body, r, eta, kind, radii, uw, points=None, bg=None, k_fib=None, defect=None):
    """the listener's velocity_field: ((ext, S, K) of velocity_at_targets, interior mask, rigid rows)"""
    return (velocity_at_targets(fib, shell, body, r, eta, points, bg, k_fib, defect),
            *interior(r, body, kind, radii, uw, defect))


# ---- the matvec's v_all -------------------------------------------------------------------------------------------
def window(fib, shell, body, ranges=None):
    """(fa, fb, sa, sb, ba, bb) node ranges of set_target_ranges' (f0, f1, s0, s1, b0, b1) (None: everything)"""
    nf, ns, nb = fib["pos"].shape[0], shell["pos"].shape[0], body["pos"].shape[0]
    if ranges is None:
        return 0, nf, 0, ns, 0, nb
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])]).astype(np.int64)
    f0, f1, s0, s1, b0, b1 = ranges
    return int(off[f0]), int(off[f1]), s0, s1, b0, b1


def matvec(fib, shell, body, eta, ranges=None, k_fib=None, rows=None, defect=None):
    """v_all of skb_flow_matvec at the rows [own fiber nodes | own shell rows | own body rows] (matvec_core), or at
    `rows` of that list:
        fiber rows   fibers' pairs - self term + periphery + bodies
        shell rows   fibers' pairs + bodies
        body rows    fibers' pairs + periphery + bodies
    k_fib: the symmetric kernel's K of the fiber pairs at the fiber rows (scalar), when it can run"""
    fa, fb, sa, sb, ba, bb = window(fib, shell, body, ranges)
    nf = fib["pos"].shape[0]
    has_f, has_s = nf > 0, shell["pos"].shape[0] > 0
    wf = ps.weighted_forces(fib["forces"], fiber_weights(fib, defect)) if has_f else None
    n_win = (fb - fa) + (sb - sa) + (bb - ba)
    rows = np.arange(n_win) if rows is None else np.asarray(rows, dtype=np.int64)
    blocks, lo = [], 0
    for cls, tr in (("f", fib["pos"][fa:fb]), ("s", shell["pos"][sa:sb]), ("b", body["pos"][ba:bb])):
        sel = rows[(rows >= lo) & (rows < lo + len(tr))] - lo
        lo += len(tr)
        if sel.size == 0:
            continue
        tr = tr[sel]
        parts = []
        if has_f:
            parts.append(fiber_pairs(fib, tr, eta, k_fib if cls == "f" else None, defect))
        if cls == "f":
            nodes = fa + sel
            if defect == "self_window_offset":
                nodes = np.where(sel >= fa, sel, -1)
            st = self_term(fib["pos"], fib["n_nodes"], wf, eta, nodes, defect)
            if defect in ("self_twice", "self_skipped"):
                st = (st[0] * (2 if defect == "self_twice" else 0), st[1], st[2])
            parts.append(st)
        if has_s and cls != "s":
            parts.append(periphery_flow(shell, tr, eta, defect=defect))
        parts += body_flow(body, tr, eta, defect)
        if parts:
            blocks.append(compose(*parts))
        else:
            z = np.zeros((len(tr), 3), dtype=LD)
            blocks.append((z, z.copy(), np.zeros(len(tr))))
    if not blocks:
        z = np.zeros((0, 3), dtype=LD)
        return z, z.copy(), np.zeros(0)
    return concat(*blocks)

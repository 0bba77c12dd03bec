"""Extended-precision restatement of skb_flow_listener_gradient, the velocity gradient and pressure of the listener's
frame (skb_matvec.cu gradient_dev; skb_runtime.cu Evaluator::gradient; pair_kernels.cuh stokeslet_grad_source,
stresslet_grad_source; aux_kernels.cuh oseen_grad_add_kernel, rotlet_grad_add_kernel, background_grad_add_kernel;
listener_kernels.cuh gradient_finish_kernel) -- TEST INFRASTRUCTURE ONLY.  Conventions of tests/flow_reference.py and
tests/pair_sum_reference.py (U, ratio, compose): every function takes float64 inputs and returns, per target row and for
each of the 10 outputs (d u_i / d x_j at 3 i + j, then the pressure), (ext, S, K):

    ext  in np.longdouble, the function of the float64 inputs the device computes, with the device's own rules;
    S    the same computation on absolute values, every signed sub-term taken separately;
    K    (per row) the worst-case rounding count of the device's evaluation, fixed from the kernel source below.

A device output passes when |dev - ext| <= K u S, u = 2^-53.  r = x_trg - x_src throughout, c = 1 / (8 pi eta).

What is restated.
    Stokeslet (the fibers' trapezoid-weighted forces, the bodies' centre forces; packed strengths bit for bit in
    float64, pair_sum_reference.weighted_forces):
        G_ij = d_i f_j y^3 - 3 d_i d_j (f.d) y^5 - f_i d_j y^3 + delta_ij (f.d) y^3,   p / eta = 2 (f.d) y^3,
        post-scaled by c.
    stresslet (the periphery and the body surfaces: 2 eta n (x) rho through its sym6 w, double_layer_sym6):
        A = d.S.d, h = 2 S_sym d,  G_ij = d_i h_j y^5 - 5 A y^7 d_i d_j + delta_ij A y^5,
        p / eta = 2 A y^5 - (2/3) tr(S) y^3, post-scaled by -3 c.
    Oseen (point forces, oseen_grad_add_kernel): the Stokeslet's G and p with 1 / D for y, scaled by c.
    rotlet (point torques and the bodies' centre torques, rotlet_grad_add_kernel): m = L x d,
        G_ij = c (eps_iaj L_a / D^3 - 3 m_i d_j / D^5), no pressure.
    background: scale_j at (j, c_j).
    gradient_finish_kernel: the pressure times eta; rows some body's interior test takes (kind != 0; the last such
        body wins) hold that body's rigid gradient, eps_ikj omega_k, bitwise, and a NaN pressure.

Branch rules, each decided on the float64 value the kernel forms, never on the exact one:
    pair kernels      a pair adds exactly 0 when the kernel's r^2 -- d rounded, then dx*dx, fma(dy, dy, .), fma(dz, dz,
                      .), written as explicit fma in rsqrt_or_zero's callers -- is below DBL_MIN (r == 0 and subnormal
                      r^2: the seed instruction flushes those).  The padded odd source of the gradient kinds' last tile
                      has zero strength and adds exactly 0.
    Oseen             skipped when the float64 r = sqrt(r^2) == 0; regularised, D = sqrt(r^2 + REG2), when r <= EPS.
    rotlet            skipped when the float64 r^2 == 0; regularised, D = sqrt(REG2 + r^2), when r^2 < EPS2, with
                      EPS2 = kEps * kEps rounded.  (The rotlet velocity has no such skip; its regularised gradient at
                      r = 0 would be c eps_iaj L_a / REG^3, so the skip is a rule of its own.)
    The aux kernels' r^2 = d0 d0 + d1 d1 + d2 d2 is left to nvcc: the built library (skellysim_b200/csrc/Makefile:
    nvcc -O3 -gencode arch=compute_90a,code=sm_90a, FMA contraction at its default, no fast-math; read with
    cuobjdump -sass) forms it in both oseen_grad_add_kernel and rotlet_grad_add_kernel as DMUL then two DFMA, the
    contracted form pair_sum_reference.r2_kernel computes.  Each decision is still taken on both the contracted and the
    plain form and a geometry where they disagree is refused (ValueError, flow_reference._decide), so no test depends
    on the build's choice.  Axis-aligned offsets (dy = dz = 0) make every form exact.

K (first-order counts in u, an FMA counts one, relative to the sub-term's absolute value; psi = 8 is the error of
y = 1/|d| from pair_sum_reference, the same seed and third-order step):
    K_PAIR_GRAD["sl"] -- stokeslet_grad_source, one pair, its own roundings into the accumulators included:
        d 1;  r^2 5;  y psi = 8;  y2 = y y: 17;  y3 = y2 y: 26;  f.d: 4;  a = (f.d) y3: 31
        b = (3 a) y2: 32 + 17 + 1 = 50;  q_j = d_j y3: 28;  p_j = fma(-d_j, b, f_j y3): 1 + 50 + 1 = 52
        g_ij = fma(-f_i, q_j, fma(d_i, p_j, g)): 1 + 52 + 1 + 1 = 55;  diagonal g += a: 56
        pressure fma(2, a, g): 32                                                                           56
    K_PAIR_GRAD["dl6"] -- stresslet_grad_source:
        y3 26;  y5 = y3 y2: 44;  h_j: d 1 + three roundings = 4;  h.d: 4 + 1 + 3 = 8
        A5 = (0.5 (h.d)) y5: 8 + 44 + 1 = 53;  c5 = (5 A5) y2: 54 + 17 + 1 = 72
        v_j = fma(-c5, d_j, h_j y5): 1 + 72 + 1 = 74;  g_ij = fma(d_i, v_j, g): 76;  diagonal g += A5: 77
        pressure: tr23 = (2/3)(w0 + w1 + w2): 4;  fma(2, A5, fma(-tr23, y3, g)): max(4 + 26 + 2, 53 + 1) = 54      77
    K_depth -- every rounding a term passes after its own pair: each later source adds to the worst output's running
        sum ADDS roundings (Stokeslet diagonal: two FMAs and the += of a, 3; stresslet diagonal and pressure, 2), over
        at most ceil(n_src / 128) 128 sources of one split, then reduce_partials adds at most min(tiles, 256) split
        partials.  The gradient kinds' plan is not observable (skb_plan_query refuses kinds 2 and 3), so this is
        pair_sum_reference's upper bound for an unobservable plan with the walk scaled by ADDS:
        ADDS ceil(n_src / 128) 128 + min(tiles, 256).
    K_SCALE = 5 -- scale_mul = 1 / eta (1), (1 | -3) / (8 M_PI) (2), their product (1), the post-scale multiply (1).
    K_OSEEN_GRAD_PAIR -- oseen_grad_add_kernel, one pair, its += into a[] and c's error included:
        d 1;  r^2 5;  r = sqrt: 3.5;  regularised D: r r 8, + REG2 (REG2 rounded) 9, sqrt 5.5 (unregularised 3.5)
        D D: 12;  D D D: 18.5;  gr = 1 / (D D D): 19.5;  hr = (3 gr) / (D D): 20.5 + 12 + 1 = 33.5;  r.f: 4
        delta_ij r.f + d_i f_j - f_i d_j: 6;  gr (.): 26.5;  ((hr r.f) d_i) d_j: 33.5 + 4 + 1 + 2 + 2 = 42.5
        their difference 43.5;  a += : 44.5;  pressure (2 gr) r.f: 24.5 + 1
        c = 1 / (8 M_PI eta): 3;  c a: 1                                                                   49
    K_ROTLET_GRAD_PAIR -- rotlet_grad_add_kernel:
        d 1;  r^2 5;  D: sqrt(r^2) 3.5 or sqrt(REG2 + r^2) 4;  D D D: 14;  fr = 1 / (.): 15
        hr = (3 fr) / (D D): 16 + 9 + 1 = 26;  m_i = d_b L_c - d_c L_b: 3;  fr e_ij: 16
        (hr m_i) d_j: 26 + 3 + 1 + 2 = 32;  difference 33;  a += : 34;  c 3, c a 1                           38
    k_points(m) = K_OSEEN_GRAD_PAIR + m (the sum over the sources) + K_REF(4 m) + SLACK, k_rotlet(m) likewise with
    K_ROTLET_GRAD_PAIR and K_REF(2 m); K_BG = 0 (its one rounding is the accumulate compose counts).
    k_pair(kind, n) = K_PAIR_GRAD[kind] + K_depth + K_SCALE + K_REF(4 n) + SLACK.
    K_REF(N) = pair_sum_reference.k_ref of the N sub-terms summed in long double;  SLACK = 4 (second-order terms and the
    double rounding of an FMA emulated in long double).
    A row composes its parts (flow_reference.compose): the largest K of its parts plus one for each part's accumulate
    into g, plus K_ETA = 1 for gradient_finish_kernel's multiply of the pressure by eta (counted on every output).

Domain.  The bound holds where every y^k a chain forms stays a normal float64: y^5 for the Stokeslet gradient, y^7 (as
y5 y2) for the stresslet gradient, so separations from about 1e-40 to 1e40 for unit-sized strengths.  Nothing is
asserted outside it: at r^2 = DBL_MIN exactly y^3 = 2^1533 overflows, so of the two sides of DBL_MIN only the masked one
(r^2 below it, the pair exactly 0) is in the domain.

Planted defects (defect=), each a slip the kernels or their composition could make;
tests/test_listener_gradient_ext_cpu.py shows that each misses its bound by more than 1e9 K on some row:
    oseen_r_for_D        the Oseen gradient's 1 / D^5 formed with r for D: hr = 3 gr / (r r)
    oseen_eps_strict     dr >= eps in place of dr > eps (the row at float64 r == EPS unregularised)
    rotlet_r0_kept       the rotlet gradient's r^2 == 0 skip removed
    rotlet_eps_le        the rotlet regularises at r^2 <= EPS2
    no_subnormal_rule    the pair kinds evaluate pairs whose float64 r^2 is subnormal
    tr_dropped           the stresslet pressure's -(2/3) tr(S) y^3 dropped
    pressure_no_eta      the pressure not multiplied by eta
    fr_transposed        -f_i r_j written -f_j r_i
    ragged_tile_dropped  the pair kinds' ragged last source tile dropped
    split_dropped        the reduce leaves out the last split's partial (plan= (tiles_per_split, n_splits), default the
                         upper-bound plan)
    bg_component         the background's component map ignored: scale_j at (j, j)
"""
import numpy as np

import flow_reference as fr
import pair_sum_reference as ps
from body_block_reference import U, ratio  # noqa: F401  (for the tests)

LD = np.longdouble
EPS, REG, REG2, EPS2 = fr.EPS, fr.REG, fr.REG2, fr.EPS2
SLACK = 4
K_PAIR_GRAD = {"sl": 56, "dl6": 77}
ADDS = {"sl": 3, "dl6": 2}
K_SCALE = ps.K_SCALE
K_OSEEN_GRAD_PAIR = 49
K_ROTLET_GRAD_PAIR = 38
K_BG = 0
K_ETA = 1
NOUT = 10

DEFECTS = ("oseen_r_for_D", "oseen_eps_strict", "rotlet_r0_kept", "rotlet_eps_le", "no_subnormal_rule", "tr_dropped",
           "pressure_no_eta", "fr_transposed", "ragged_tile_dropped", "split_dropped", "bg_component")

_EYE = np.eye(3, dtype=LD)
_LEVI = np.zeros((3, 3, 3), dtype=LD)
for _i, _a, _j in ((0, 1, 2), (1, 2, 0), (2, 0, 1)):
    _LEVI[_i, _a, _j], _LEVI[_i, _j, _a] = 1, -1


# ---- K ------------------------------------------------------------------------------------------------------------
def bound_plan(n_src):
    """(tiles_per_split, n_splits) of the upper-bound plan: one source tile per split, at most 256 splits"""
    tiles = -(-n_src // ps.SRC_TILE)
    s = min(tiles, ps.MAX_SPLITS)
    return -(-tiles // s), s


def k_pair(kind, n_src):
    tiles = -(-n_src // ps.SRC_TILE)
    depth = ADDS[kind] * tiles * ps.SRC_TILE + min(tiles, ps.MAX_SPLITS)
    return K_PAIR_GRAD[kind] + depth + K_SCALE + ps.k_ref(4 * n_src) + SLACK


def k_points(m):
    return K_OSEEN_GRAD_PAIR + m + ps.k_ref(4 * m) + SLACK


def k_rotlet(m):
    return K_ROTLET_GRAD_PAIR + m + ps.k_ref(2 * m) + SLACK


# ---- pair kinds ---------------------------------------------------------------------------------------------------
def _out(G, P):
    """(..., 3, 3) and (...,) -> (..., 10)"""
    return np.concatenate([G.reshape(G.shape[:-2] + (9,)), P[..., None]], axis=-1)


def grad_terms(kind, d, keep, f, fa, defect=None):
    """(term, aterm) (..., 10), unscaled, of the pairs with long-double differences d (..., 3), the kernel's mask and
    signed / absolute strengths f, fa (..., 3 Stokeslet or ..., 6 sym6)"""
    r2 = (d * d).sum(axis=-1)
    y = np.where(keep, 1 / np.sqrt(np.where(keep, r2, LD(1))), LD(0))
    y3, y5 = y ** 3, y ** 5
    a = np.abs(d)
    di, dj = d[..., :, None], d[..., None, :]
    ai, aj = a[..., :, None], a[..., None, :]
    E = _EYE
    if kind == "sl":
        fd, fad = (f * d).sum(axis=-1), (fa * a).sum(axis=-1)
        fi, fj = f[..., :, None], f[..., None, :]
        Fi, Fj = fa[..., :, None], fa[..., None, :]
        t3, t5 = y3[..., None, None], y5[..., None, None]
        minus_fr = fj * di if defect == "fr_transposed" else fi * dj
        G = di * fj * t3 - 3 * di * dj * (fd * y5)[..., None, None] - minus_fr * t3 + E * (fd * y3)[..., None, None]
        SG = ai * Fj * t3 + 3 * ai * aj * (fad * y5)[..., None, None] + Fi * aj * t3 + E * (fad * y3)[..., None, None]
        return _out(G, 2 * fd * y3), _out(SG, 2 * fad * y3)
    y7 = y5 * y * y
    pd = (d[..., 0] ** 2, d[..., 1] ** 2, d[..., 2] ** 2, d[..., 0] * d[..., 1], d[..., 0] * d[..., 2],
          d[..., 1] * d[..., 2])
    pa = (a[..., 0] ** 2, a[..., 1] ** 2, a[..., 2] ** 2, a[..., 0] * a[..., 1], a[..., 0] * a[..., 2],
          a[..., 1] * a[..., 2])
    A = sum(f[..., k] * pd[k] for k in range(6))
    Aa = sum(fa[..., k] * pa[k] for k in range(6))

    def hvec(w, v):
        return np.stack([2 * w[..., 0] * v[..., 0] + w[..., 3] * v[..., 1] + w[..., 4] * v[..., 2],
                         w[..., 3] * v[..., 0] + 2 * w[..., 1] * v[..., 1] + w[..., 5] * v[..., 2],
                         w[..., 4] * v[..., 0] + w[..., 5] * v[..., 1] + 2 * w[..., 2] * v[..., 2]], axis=-1)
    h, ha = hvec(f, d), hvec(fa, a)
    t5 = y5[..., None, None]
    G = di * h[..., None, :] * t5 - 5 * di * dj * (A * y7)[..., None, None] + E * (A * y5)[..., None, None]
    SG = ai * ha[..., None, :] * t5 + 5 * ai * aj * (Aa * y7)[..., None, None] + E * (Aa * y5)[..., None, None]
    tr, tra = f[..., 0] + f[..., 1] + f[..., 2], fa[..., 0] + fa[..., 1] + fa[..., 2]
    trw = LD(0) if defect == "tr_dropped" else LD(1)
    return _out(G, 2 * A * y5 - trw * (2 * tr / 3) * y3), _out(SG, 2 * Aa * y5 + (2 * tra / 3) * y3)


def pair_keep(d64, defect=None):
    """the pair kinds' mask on the kernel's float64 r^2 (explicit FMAs: no contraction question)"""
    r2k = ps.r2_kernel(d64[..., 0], d64[..., 1], d64[..., 2])
    return r2k > 0 if defect == "no_subnormal_rule" else r2k >= ps.DBL_MIN


def pair_grad_ext(kind, t, s, f):
    """(ext, S) (N, 10), unscaled, of N single pairs (t[k], s[k], f[k])"""
    t, s, f = (np.asarray(x, dtype=np.float64) for x in (t, s, f))
    fl = f.astype(LD)
    return grad_terms(kind, t.astype(LD) - s.astype(LD), pair_keep(t - s), fl, np.abs(fl))


def _source_keep(n, defect, plan):
    keep = np.ones(n, dtype=bool)
    if defect == "ragged_tile_dropped":
        keep[(n // ps.SRC_TILE) * ps.SRC_TILE:] = False
    elif defect == "split_dropped":
        per, n_splits = bound_plan(n) if plan is None else plan
        keep[(n_splits - 1) * per * ps.SRC_TILE:] = False
    return keep


def pair_grad_rows(kind, r_src, f_src, r_trg, eta, defect=None, plan=None, chunk=1 << 16):
    """(ext, S, K) of the gradient kind of `kind` ("sl": packed Stokeslet strengths (n, 3); "dl6": packed sym6 (n, 6))
    at every target, post-scaled by (1 | -3) c"""
    r_src = np.asarray(r_src, dtype=np.float64).reshape(-1, 3)
    r_trg = np.asarray(r_trg, dtype=np.float64).reshape(-1, 3)
    f_src = np.asarray(f_src, dtype=np.float64).reshape(len(r_src), -1)
    n = len(r_src)
    sel = _source_keep(n, defect, plan)
    ext = np.zeros((len(r_trg), NOUT), dtype=LD)
    S = np.zeros((len(r_trg), NOUT), dtype=LD)
    step = max(1, chunk // max(n, 1))
    fl = f_src.astype(LD)
    for a in range(0, len(r_trg), step):
        t = r_trg[a:a + step]
        d64 = t[:, None, :] - r_src[None, :, :]
        keep = pair_keep(d64, defect) & sel[None, :]
        d = t.astype(LD)[:, None, :] - r_src.astype(LD)[None, :, :]
        term, aterm = grad_terms(kind, d, keep, fl[None], np.abs(fl)[None], defect)
        ext[a:a + step], S[a:a + step] = term.sum(axis=1), aterm.sum(axis=1)
    sc = ps.scale_of(kind, eta)
    return fr.part(ext * sc, S * abs(sc), k_pair(kind, n))


# ---- the aux kernels ----------------------------------------------------------------------------------------------
def oseen_grad(r_trg, pts, forces, eta, defect=None):
    """oseen_grad_add_kernel at every target: (ext, S, K)"""
    t, s = np.asarray(r_trg, dtype=np.float64), np.asarray(pts, dtype=np.float64)
    d64 = t[:, None, :] - s[None, :, :]

    def rule(r2):
        r = np.sqrt(r2)
        return r == 0.0, (r < EPS) if defect == "oseen_eps_strict" else (r <= EPS)
    skip, reg = fr._decide(d64, rule)
    d = t.astype(LD)[:, None, :] - s.astype(LD)[None, :, :]
    r2 = (d * d).sum(axis=-1)
    D2 = np.where(skip, LD(1), np.where(reg, r2 + LD(REG2), r2))
    y3 = np.where(skip, LD(0), D2 ** LD(-1.5))
    D2h = np.where(reg & (defect == "oseen_r_for_D"), np.where(skip, LD(1), r2), D2)
    y5 = y3 / D2h
    F = np.asarray(forces, dtype=np.float64).astype(LD)[None]
    Fa, a = np.abs(F), np.abs(d)
    fd, fad = (F * d).sum(axis=-1), (Fa * a).sum(axis=-1)
    di, dj, ai, aj = d[..., :, None], d[..., None, :], a[..., :, None], a[..., None, :]
    t3 = y3[..., None, None]
    G = t3 * (_EYE * fd[..., None, None] + di * F[..., None, :] - F[..., :, None] * dj) \
        - 3 * (y5 * fd)[..., None, None] * di * dj
    SG = t3 * (_EYE * fad[..., None, None] + ai * Fa[..., None, :] + Fa[..., :, None] * aj) \
        + 3 * (y5 * fad)[..., None, None] * ai * aj
    c = fr.c_of(eta)
    return fr.part(c * _out(G, 2 * fd * y3).sum(axis=1), c * _out(SG, 2 * fad * y3).sum(axis=1), k_points(len(s)))


def rotlet_grad(r_trg, src, torques, eta, defect=None):
    """rotlet_grad_add_kernel at every target: (ext, S, K)"""
    t, s = np.asarray(r_trg, dtype=np.float64), np.asarray(src, dtype=np.float64)
    d64 = t[:, None, :] - s[None, :, :]
    skip, reg = fr._decide(d64, lambda r2: (np.zeros(r2.shape, dtype=bool) if defect == "rotlet_r0_kept"
                                            else r2 == 0.0,
                                            (r2 <= EPS2) if defect == "rotlet_eps_le" else (r2 < EPS2)))
    d = t.astype(LD)[:, None, :] - s.astype(LD)[None, :, :]
    r2 = (d * d).sum(axis=-1)
    D2 = np.where(reg, r2 + LD(REG2), r2)
    live = ~skip & (D2 > 0)
    D2 = np.where(live, D2, LD(1))
    y3 = np.where(live, D2 ** LD(-1.5), LD(0))
    y5 = y3 / D2
    L = np.asarray(torques, dtype=np.float64).astype(LD)[None]
    La, a = np.abs(L), np.abs(d)
    m = np.cross(L, d)
    ma = np.stack([La[..., 1] * a[..., 2] + La[..., 2] * a[..., 1], La[..., 2] * a[..., 0] + La[..., 0] * a[..., 2],
                   La[..., 0] * a[..., 1] + La[..., 1] * a[..., 0]], axis=-1)
    E = np.einsum("iaj,...a->...ij", _LEVI, L)
    G = y3[..., None, None] * E - 3 * y5[..., None, None] * m[..., :, None] * d[..., None, :]
    SG = y3[..., None, None] * np.abs(E) + 3 * y5[..., None, None] * ma[..., :, None] * a[..., None, :]
    z = np.zeros(G.shape[:-2], dtype=LD)
    c = fr.c_of(eta)
    return fr.part(c * _out(G, z).sum(axis=1), c * _out(SG, z).sum(axis=1), k_rotlet(len(s)))


def background_grad(n_trg, comp, scale, defect=None):
    """background_grad_add_kernel: (ext, S, K)"""
    comp = [0, 1, 2] if defect == "bg_component" else [int(c) for c in comp]
    g = np.zeros(NOUT, dtype=LD)
    for j in range(3):
        g[3 * j + comp[j]] += LD(np.float64(scale[j]))
    g = np.broadcast_to(g, (n_trg, NOUT))
    return fr.part(g, np.abs(g), K_BG + SLACK)


# ---- the frame ----------------------------------------------------------------------------------------------------
def frame(fib, shell, body, r, eta, points=None, bg=None, defect=None, plan=None):
    """gradient_dev then gradient_finish_kernel's multiply of the pressure by eta, at every row as a fluid point:
    fibers, body surfaces, body centre forces and torques, periphery, point forces and torques, background"""
    r = np.asarray(r, dtype=np.float64).reshape(-1, 3)
    parts = []
    if len(fib["pos"]):
        wf = ps.weighted_forces(fib["forces"], fr.fiber_weights(fib))
        parts.append(pair_grad_rows("sl", fib["pos"], wf, r, eta, defect, plan))
    if len(body["centers"]):
        if len(body["pos"]):
            s6 = ps.double_layer_sym6(body["normals"], body["density"], eta)
            parts.append(pair_grad_rows("dl6", body["pos"], s6, r, eta, defect, plan))
        parts.append(pair_grad_rows("sl", body["centers"], body["forces"], r, eta, defect, plan))
        parts.append(rotlet_grad(r, body["centers"], body["torques"], eta, defect))
    if len(shell["pos"]):
        s6 = ps.double_layer_sym6(shell["normals"], shell["density"], eta)
        parts.append(pair_grad_rows("dl6", shell["pos"], s6, r, eta, defect, plan))
    if points is not None and len(points[0]):
        pts, pf, ptq = points
        parts += [oseen_grad(r, pts, pf, eta, defect), rotlet_grad(r, pts, ptq, eta, defect)]
    if bg is not None:
        parts.append(background_grad(len(r), bg[0], bg[1], defect))
    if not parts:
        z = np.zeros((len(r), NOUT), dtype=LD)
        return z, z.copy(), np.full(len(r), float(K_ETA))
    ext, S, K = fr.compose(*parts)
    if defect != "pressure_no_eta":
        ext[:, 9] *= LD(np.float64(eta))
        S[:, 9] *= LD(np.float64(eta))
    return ext, S, K + K_ETA


def rigid_gradient(omega):
    """the rigid motion's gradient eps_ikj omega_k (row-major) and a NaN pressure, as gradient_finish_kernel writes
    it"""
    w0, w1, w2 = (np.float64(x) for x in omega)
    return np.array([0.0, -w2, w1, w2, 0.0, -w0, -w1, w0, 0.0, np.nan])


def interior(r, body, kind, radii, uw):
    """(mask, rigid (n, 10)) of gradient_finish_kernel: the rows some body's interior test takes, and there the last
    such body's rigid gradient and a NaN pressure (the test of flow_reference.interior, bodies in order)"""
    r = np.asarray(r, dtype=np.float64).reshape(-1, 3)
    mask = np.zeros(len(r), dtype=bool)
    out = np.zeros((len(r), NOUT))
    for b in range(len(body["centers"])):
        m, _ = fr.interior(r, dict(centers=np.asarray(body["centers"])[b:b + 1]), np.asarray(kind)[b:b + 1],
                           np.asarray(radii)[b:b + 1], np.asarray(uw)[b:b + 1])
        out[m] = rigid_gradient(np.asarray(uw)[b][3:])
        mask |= m
    return mask, out


def listener_gradient(fib, shell, body, r, eta, kind, radii, uw, points=None, bg=None, defect=None):
    """((ext, S, K) of frame, interior mask, rigid rows)"""
    return (frame(fib, shell, body, r, eta, points, bg, defect), *interior(r, body, kind, radii, uw))


def as_grad_pressure(x):
    """(n, 10) -> (G (n, 3, 3), p (n,))"""
    x = np.asarray(x)
    return x[:, :9].reshape(-1, 3, 3), x[:, 9]


# ---- one pair in the kernels' float64 instruction order -------------------------------------------------------------
def add_pair_f64(kind, g, t, s, f, seed_err):
    """g (N, 10) float64 after the gradient kind's chain adds the pairs (t[k], s[k], f[k]) into it, every instruction
    in stokeslet_grad_source's / stresslet_grad_source's order, the rsqrt seed's relative error `seed_err`"""
    fma = ps.fma
    t, s, f = (np.asarray(x, dtype=np.float64) for x in (t, s, f))
    g = np.array(g, dtype=np.float64, copy=True)
    with np.errstate(over="ignore", invalid="ignore"):
        d = t - s
        r2 = ps.r2_kernel(d[:, 0], d[:, 1], d[:, 2])
        y = ps._rsqrt(r2, seed_err, None)
        y2 = y * y
        y3 = y2 * y
        if kind == "sl":
            a = fma(f[:, 2], d[:, 2], fma(f[:, 1], d[:, 1], f[:, 0] * d[:, 0])) * y3
            b = (3.0 * a) * y2
            q = [d[:, j] * y3 for j in range(3)]
            p = [fma(-d[:, j], b, f[:, j] * y3) for j in range(3)]
            for i in range(3):
                for j in range(3):
                    g[:, 3 * i + j] = fma(-f[:, i], q[j], fma(d[:, i], p[j], g[:, 3 * i + j]))
            for i in range(3):
                g[:, 4 * i] = g[:, 4 * i] + a
            g[:, 9] = fma(2.0, a, g[:, 9])
            return g
        w = f
        tr23 = (2.0 / 3.0) * ((w[:, 0] + w[:, 1]) + w[:, 2])
        y5 = y3 * y2
        h = [fma(2.0 * w[:, 0], d[:, 0], fma(w[:, 3], d[:, 1], w[:, 4] * d[:, 2])),
             fma(w[:, 3], d[:, 0], fma(2.0 * w[:, 1], d[:, 1], w[:, 5] * d[:, 2])),
             fma(w[:, 4], d[:, 0], fma(w[:, 5], d[:, 1], (2.0 * w[:, 2]) * d[:, 2]))]
        A5 = (0.5 * fma(h[2], d[:, 2], fma(h[1], d[:, 1], h[0] * d[:, 0]))) * y5
        c5 = (5.0 * A5) * y2
        v = [fma(-c5, d[:, j], h[j] * y5) for j in range(3)]
        for i in range(3):
            for j in range(3):
                g[:, 3 * i + j] = fma(d[:, i], v[j], g[:, 3 * i + j])
        for i in range(3):
            g[:, 4 * i] = g[:, 4 * i] + A5
        g[:, 9] = fma(2.0, A5, fma(-tr23, y3, g[:, 9]))
        return g

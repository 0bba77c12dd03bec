"""Extended-precision restatement of the all-pairs Stokeslet / stresslet sums of pair_sum_kernel (pair_kernels.cuh), the
symmetric kernel pair_sym_kernel (sym_kernels.cuh) and the fiber-periphery cross kernel pair_cross_kernel
(cross_kernels.cuh) -- TEST INFRASTRUCTURE ONLY.  Conventions of tests/body_block_reference.py (U, ratio).

pair_blocks() / pair_rows() take float64 inputs and return, for the requested target rows, in np.longdouble:

    ext  the function of the float64 inputs the kernels compute, with the kernels' own rules:
         * r == 0 rule: a pair contributes exactly 0 when the kernel's float64 r^2 -- dx = t - s rounded, then
           dx*dx, fma(dy, dy, .), fma(dz, dz, .) -- is below DBL_MIN = 2^-1022 (r == 0 and subnormal r^2: the seed
           instruction flushes those; DESIGN §5).  The mask is decided on that float64 r^2, never on the exact one.
         * fused exclusion: a pair whose target and source carry the same fiber id contributes exactly 0 (only the
           leading targets carry ids; the others carry -1).
         * Stokeslet  u = 1/(8 pi) sum_j y (f_j + d (f_j . d) y^2),     d = t - s_j, y = 1/|d|
           stresslet  u = -3/(8 pi) sum_j d (d . S_j . d) y^5,        S_j entering through its sym6 contraction
                      (sxx, syy, szz, sxy + syx, sxz + szx, syz + szy).
         * packed strengths the device forms in float64 before the pair sums are restated bit for bit in float64 and
           are then exact inputs: the trapezoid weights of fiber_weights_kernel, 0.5 L (w0 / (n - 1)), and the weighted
           forces f w (pack_sl_kernel); the double layer's sym6 of pack_dl_normal_density_kernel, n' = (2 eta) n, then
           n'_a rho_a and n'_a rho_b + n'_b rho_a, every product and sum rounded once (no contraction).
    S    the error scale: the same sum with every input by its absolute value, every difference of coordinates as |d|
         (one rounded subtraction errs by u relative to its result), and every signed sum a sum of absolute values
         (r.S.r term by term, sxy + syx as |sxy| + |syx|, f.d as |f|.|d|).

Rows are evaluated against the sources in chunks, so memory stays bounded.

The criterion.  A device row passes when |dev - ext| <= K u S component by component, u = 2^-53.  K counts roundings to
first order, for ANY summation tree, and is fixed from the kernel source:

K_pair -- the error of one pair's term relative to that pair's absolute term, the pair's own accumulate included.
    Each line below is an error relative to the quantity named, in units of u (an FMA rounds once).
    d_k = t_k - s_k                                  1
    r^2: d_k rounded (2) + dx*dx, two fma (3)         5   (all terms positive)
    y = 1/|d|: half of r^2's                        2.5
        seed y0 (MUFU.RSQ64H, rel. error <= 2^-22.4) then ONE third-order step, h = e (1/2 + 3/8 e), e = 1 - r^2 y0^2:
        residual (5/16) e^3 <= (5/16) (2^-21.4)^3 < 2^-65.8 = 0.0003 u; the step's five roundings (r^2 y0, the fma
        forming e, the fma forming 1/2 + 3/8 e, the product h, the fma y0 + y0 h) counted as 1 each            5
        -> psi, the error of y                         8   (7.5 + residual, rounded up)
    Stokeslet (stokeslet_chains, stokeslet_pairpairs, cross_pairpairs' reverse direction):
        f.d: d rounded (1), product and two fma (3)                                       4
        y^2: 2 psi + 1 = 17;  q = (f.d) y^2: 4 + 17 + 1                                  22
        v_k = fma(d_k, q, f_k): on the d-term 1 + 22 + 1, on the f-term 1                 24
        y v_k: psi more on both terms                                                     32
        the accumulate into the running sum                                               1
        K_PAIR_SL                                                                         33
    stresslet (stresslet_chains, cross_pairpairs' forward direction), r.S.r in the kernels' order
        (sxx dx + pxy dy + pxz dz) dx + (syy dy + pyz dz) dy + (szz dz) dz, d rounded on every factor:
        deepest term 8;  sym6 sums sxy + syx from raw 9-component strengths, 1                 9
        y^5 = ((y y)(y y)) y: 5 psi + 3 roundings                                          43 (counted 44)
        co = (r.S.r) y^5: 9 + 44 + 1                                                       54
        d_k co: d_k rounded                                                                55
        the accumulate                                                                      1
        K_PAIR_DL                                                                          56
K_depth -- every addition a term passes after its own accumulate, on its way to the row (a term's path in any
    summation tree is at most the tree's depth, and adding an exact zero -- a padded source, a masked pair -- is exact):
    plain kernel      min(tiles_per_split * 128, n_src + 1) (the running sums of one split, two sources per step, the
                      padded odd source an exact zero) + n_splits (reduce_partials_kernel / reduce_partials_wide_kernel, any
                      order), from the plan the call used (Context.stats(), capi.plan_query for the same arguments).
                      When the plan is not observable (the remainder targets of the symmetric path, the periphery rows
                      of a matvec without the cross kernel): its upper bound ceil(n_src / 128) * 128 + min(tiles, 256).
    symmetric kernel  n_pad (a forward partial walks at most every node of the padded list; a reverse partial 256 = 32
                      lanes x 8 targets) + 3 (the four warps' slabs) + the partials sym_reduce_kernel adds into a row of
                      block b: the owned rows I < b of P plus the items of row b (capi.sym_plan_query) + 1.
    cross kernel      fiber rows: an item's running sum walks at most every periphery node (n_sh rounded up to 32), then
                      cross_reduce_fib_kernel adds the block's items (at most one per 32-node group); periphery rows:
                      the ring's 128 = 32 lanes x 4 targets, 3 slab adds, then cross_reduce_shell_kernel adds one
                      partial per 512-node fiber block.  Both within n_src rounded up to 32 + ceil(n_src / 32) + 4.
K_SCALE = 5 -- the post-scale multiply (1) and the scale constant, -3.0 / (8.0 * M_PI * eta) and its relatives: M_PI
    rounded and at most three more rounded operations (4).
K_REF -- the reference's own error: every term to 2^-64 relative and the long-double sum of N terms, N 2^-64 = N 2^-11 u,
    counted as ceil((N + 64) 2^-11) + 1.
SLACK = 4 -- second-order terms (all below 1e-6 u at these depths) and the double rounding of an FMA emulated in long
    double (< 2^-10 u per operation, tests/test_pair_sum_ext_cpu.py).

K = K_pair + K_depth + K_SCALE + K_REF + SLACK.  These are worst-case counts: no sqrt(N) or other statistical factor.

Planted defects (defect=), each a slip the kernels or their host planning could make:

    newton2              the rsqrt step second-order (h = e / 2): residual (3/8) e^2, up to ~450 u per y -- the only
                         defect that can hide inside a sum's K, so it is caught only on single-pair rows (n_src <= 2);
                         pair_terms_f64 only
    no_subnormal_rule    pairs whose float64 r^2 is subnormal are evaluated (the mask tested only r^2 == 0)
    odd_source_dropped   the last tile walks (left >> 1) source pairs: an odd last source is lost
    ragged_tile_dropped  n_src_tiles rounded down: the whole ragged last tile is lost
    split_dropped        the reduce leaves out the last split's partial
    sym6_doubled         sxy + syx formed as 2 sxy (non-symmetric 9-component strengths expose it)
    stresslet_sign       the stresslet's post-scale +3/(8 pi)
    diag_reverse_counted the reverse partial of a block-diagonal item read by the reduce: block-diagonal pairs twice
    item_reverse_dropped one item's reverse partial left out (item= (I, g0, g1) of capi.sym_plan_query)
    serpentine_flipped   a partition's owner(I) = I mod n_parts instead of the serpentine sym_row_owner
    excl_by_position     exclusion decided from list position (runs of the first fiber's length) instead of fiber id
    cross_tail_acts      the cross kernel's tail nodes beyond n_rows keep the last node's strength and act on the
                         periphery (tail = 512 ceil(n_rows / 512) - n_rows copies)
"""
import numpy as np

from body_block_reference import U, ratio  # noqa: F401  (for the tests)

LD = np.longdouble
PI = LD("3.14159265358979323846264338327950288")
DBL_MIN = 2.0 ** -1022
SEED_REL = 2.0 ** -22.4        # relative error of the MUFU.RSQ64H seed (pair_kernels.cuh)
SRC_TILE = 128                 # kSrcTile
CTA_THREADS = 128              # kCtaThreads
MAX_SPLITS = 256               # kMaxSplits
SYM_BLOCK = 1024               # kSymThreads * kSymT
SYM_GROUP = 32                 # kSymGroup
CROSS_BLOCK = 512              # kCrossBlock
PAD_TO = 1024                  # set_sources pads every source list to a multiple of this

K_PAIR = {"sl": 33, "dl9": 56, "dl6": 56}
K_SCALE = 5
SLACK = 4

DEFECTS = ("newton2", "no_subnormal_rule", "odd_source_dropped", "ragged_tile_dropped", "split_dropped",
           "sym6_doubled", "stresslet_sign", "diag_reverse_counted", "item_reverse_dropped", "serpentine_flipped",
           "excl_by_position", "cross_tail_acts")


# ---- K ------------------------------------------------------------------------------------------------------------
def k_ref(n_src):
    return int(np.ceil((n_src + 64) * 2.0 ** -11)) + 1


def k_plain(kind, n_src, tiles_per_split, n_splits):
    """K of a row of pair_sum_kernel + its reduce, from the launch plan"""
    return K_PAIR[kind] + min(tiles_per_split * SRC_TILE, n_src + 1) + n_splits + K_SCALE + k_ref(n_src) + SLACK


def k_plain_bound(kind, n_src):
    """K of a row of the plain kernel whose plan is not observable: the largest any plan can give"""
    tiles = -(-n_src // SRC_TILE)
    return k_plain(kind, n_src, tiles, min(tiles, MAX_SPLITS))


def n_pad(n_src):
    return -(-n_src // PAD_TO) * PAD_TO


def sym_partials(n_src, part=0, n_parts=1, plan=None):
    """partials sym_reduce_kernel adds into the rows of each block b: owned rows I < b of P + the items of row b"""
    nb = n_pad(n_src) // SYM_BLOCK
    if plan is None:
        from skellysim_b200 import capi
        plan = capi.sym_plan_query(nb, part, n_parts)
    _, row_begin = plan
    owned = np.array([sym_row_owner(I, n_parts) == part for I in range(nb)])
    before = np.concatenate([[0], np.cumsum(owned)[:-1]])
    return before + np.diff(np.asarray(row_begin))


def k_sym_rows(n_src, n_trg, rows, part=0, n_parts=1, plan=None):
    """K of the given rows of the symmetric path: leading rows from the plan, remainder rows by the plain bound"""
    rows = np.asarray(rows)
    parts = sym_partials(n_src, part, n_parts, plan)
    lead = rows < n_src
    K = np.full(rows.shape, float(k_plain_bound("sl", n_src)))
    b = rows[lead] // SYM_BLOCK
    K[lead] = K_PAIR["sl"] + n_pad(n_src) + 3 + parts[b] + 1 + K_SCALE + k_ref(n_src) + SLACK
    return K


def k_cross(kind, n_src):
    """K of a row of the cross kernel (fiber rows: kind dl6, n_src periphery nodes; periphery rows: kind sl, n_src fiber
    nodes)"""
    g = -(-n_src // SYM_GROUP)
    return K_PAIR[kind] + g * SYM_GROUP + g + 4 + K_SCALE + k_ref(n_src) + SLACK


# ---- structure ----------------------------------------------------------------------------------------------------
def sym_row_owner(I, n_parts):
    """skb_sym.cu sym_row_owner: serpentine"""
    k, m = divmod(I, n_parts)
    return n_parts - 1 - m if k & 1 else m


def sym_part_mult(rows, n_src, part, n_parts, defect=None, item=None):
    """(R, nb) multiplier of the 1024-node source blocks c in part `part`'s rows: a leading row (block b) holds the
    forward sums of its own blocks (c >= b, when the part owns b) and the reverse sums from the part's earlier blocks
    (c < b, when it owns c); a remainder row holds every block.  For pair_blocks(..., block=SYM_BLOCK) and combine()."""
    rows = np.asarray(rows)
    nb = -(-n_src // SYM_BLOCK)

    def owner(I):
        if defect == "serpentine_flipped":
            return I % n_parts
        k, m = np.divmod(I, n_parts)
        return np.where(k & 1, n_parts - 1 - m, m)

    b, c = (rows // SYM_BLOCK)[:, None], np.arange(nb)[None, :]
    own_b = owner(b) == part
    m = np.where(c >= b, own_b, owner(c) == part).astype(np.float64)
    if defect == "diag_reverse_counted":
        m = m + ((c == b) & own_b)
    if defect == "item_reverse_dropped":
        I, g0, g1 = item
        g = (rows // SYM_GROUP)[:, None]
        m = np.where((g >= g0) & (g < g1) & (c == I), 0.0, m)
    return np.where((rows < n_src)[:, None], m, 1.0)


def source_select(n_src, defect, tiles_per_split=None, n_splits=None):
    """the plain kernel's source-set defects"""
    def sel(rows, srcs):
        keep = np.ones(srcs.shape, dtype=bool)
        if defect == "odd_source_dropped" and n_src % 2:
            keep = srcs != n_src - 1
        elif defect == "ragged_tile_dropped":
            keep = srcs < (n_src // SRC_TILE) * SRC_TILE
        elif defect == "split_dropped":
            keep = srcs < (n_splits - 1) * tiles_per_split * SRC_TILE
        return np.broadcast_to(keep.astype(np.float64)[None, :], (rows.size, srcs.size))
    return sel


def cross_tail_select(n_rows):
    """cross_tail_acts: the last fiber node counted 1 + (tail copies) times at the periphery"""
    tail = -(-n_rows // CROSS_BLOCK) * CROSS_BLOCK - n_rows

    def sel(rows, srcs):
        return np.broadcast_to(np.where(srcs == n_rows - 1, 1.0 + tail, 1.0)[None, :], (rows.size, srcs.size))
    return sel


# ---- packed strengths, bit for bit in float64 ---------------------------------------------------------------------
def trapezoid_weights(n_nodes, lengths):
    """fiber_weights_kernel: 0.5 * L * (w0 / (n - 1)), w0 = 2 inside, 1 at both ends"""
    out = []
    for n, L in zip(n_nodes, lengths):
        w0 = np.full(n, 2.0)
        w0[0] = w0[-1] = 1.0
        out.append(0.5 * np.float64(L) * (w0 / np.float64(n - 1)))
    return np.concatenate(out) if out else np.zeros(0)


def weighted_forces(f, w):
    """pack_sl_kernel: f * w per source"""
    return np.asarray(f, dtype=np.float64) * np.asarray(w, dtype=np.float64)[:, None]


def double_layer_sym6(normals, density, eta):
    """pack_dl_normal_density_kernel: n' = (2 eta) n; (n'_0 r_0, n'_1 r_1, n'_2 r_2, n'_0 r_1 + n'_1 r_0, ...)"""
    n = (2.0 * np.float64(eta)) * np.asarray(normals, dtype=np.float64)
    r = np.asarray(density, dtype=np.float64)
    return np.stack([n[:, 0] * r[:, 0], n[:, 1] * r[:, 1], n[:, 2] * r[:, 2], n[:, 0] * r[:, 1] + n[:, 1] * r[:, 0],
                     n[:, 0] * r[:, 2] + n[:, 2] * r[:, 0], n[:, 1] * r[:, 2] + n[:, 2] * r[:, 1]], axis=1)


def scale_of(kind, eta=1.0):
    """the exact post-scale: 1/(8 pi eta) (Stokeslet) or -3/(8 pi eta) (stresslet)"""
    return (LD(1) if kind == "sl" else LD(-3)) / (LD(8) * PI * LD(eta))


# ---- float64 arithmetic of the kernels ----------------------------------------------------------------------------
def fma(a, b, c):
    """fma in float64, emulated in long double (exact product to 2^-64, then two roundings: within 2^-10 u of the
    correctly rounded fma)"""
    return (np.asarray(a, dtype=np.float64).astype(LD) * np.asarray(b, dtype=np.float64).astype(LD)
            + np.asarray(c, dtype=np.float64).astype(LD)).astype(np.float64)


def r2_kernel(dx, dy, dz):
    """the kernels' float64 r^2 from float64 differences: dx*dx, fma(dy, dy, .), fma(dz, dz, .)"""
    return fma(dz, dz, fma(dy, dy, dx * dx))


def _sym6(f, kind, defect):
    """(signed, absolute) sym6 of the strengths in long double"""
    f = np.asarray(f, dtype=np.float64)
    if kind == "dl6":
        s = f.astype(LD)
        return s, np.abs(s)
    a = f.astype(LD)
    if defect == "sym6_doubled":
        off, aoff = (2 * a[:, 1], 2 * a[:, 2], 2 * a[:, 5]), (2 * abs(a[:, 1]), 2 * abs(a[:, 2]), 2 * abs(a[:, 5]))
    else:
        off = (a[:, 1] + a[:, 3], a[:, 2] + a[:, 6], a[:, 5] + a[:, 7])
        aoff = (abs(a[:, 1]) + abs(a[:, 3]), abs(a[:, 2]) + abs(a[:, 6]), abs(a[:, 5]) + abs(a[:, 7]))
    return (np.stack([a[:, 0], a[:, 4], a[:, 8], *off], axis=1),
            np.stack([abs(a[:, 0]), abs(a[:, 4]), abs(a[:, 8]), *aoff], axis=1))


def _terms(kind, d, keep, f, g):
    """signed and absolute pair terms from long-double differences d (..., 3), the kernels' mask and the signed /
    absolute strengths f, g (..., 3 or 6)"""
    r2 = (d * d).sum(axis=-1)
    y = np.where(keep, 1 / np.sqrt(np.where(keep, r2, LD(1))), LD(0))
    a = np.abs(d)
    if kind == "sl":
        y3 = y ** 3
        return (y[..., None] * f + d * ((f * d).sum(axis=-1) * y3)[..., None],
                y[..., None] * g + a * ((g * a).sum(axis=-1) * y3)[..., None])
    y5 = y ** 5
    prods = lambda v: (v[..., 0] * v[..., 0], v[..., 1] * v[..., 1], v[..., 2] * v[..., 2], v[..., 0] * v[..., 1],
                       v[..., 0] * v[..., 2], v[..., 1] * v[..., 2])
    pd, pa = prods(d), prods(a)
    dsd = sum(f[..., k] * pd[k] for k in range(6))
    asa = sum(g[..., k] * pa[k] for k in range(6))
    return d * (dsd * y5)[..., None], a * (asa * y5)[..., None]


def pair_terms_ext(kind, t, s, f, defect=None):
    """(ext, S) of N single pairs (t[k], s[k], f[k]), unscaled: (N, 3) each"""
    t, s = np.asarray(t, dtype=np.float64), np.asarray(s, dtype=np.float64)
    if kind == "sl":
        fs = np.asarray(f, dtype=np.float64).astype(LD)
        fa = np.abs(fs)
    else:
        fs, fa = _sym6(f, kind, defect)
    d64 = t - s
    r2k = r2_kernel(d64[:, 0], d64[:, 1], d64[:, 2])
    keep = r2k > 0 if defect == "no_subnormal_rule" else r2k >= DBL_MIN
    return _terms(kind, t.astype(LD) - s.astype(LD), keep, fs, fa)


def pair_blocks(kind, r_src, f_src, r_trg, rows=None, scale=None, *, block=None, src_ids=None, trg_ids=None,
                select=None, defect=None, chunk=1 << 19):
    """(ext, S) of the pair sum of `kind` at r_trg[rows], post-scaled by `scale` (default scale_of(kind)), each
    (len(rows), n_blocks, 3) in long double: the sums over the sources of each `block`-sized run (block None: one
    run).  kind "sl": packed Stokeslet strengths (n, 3); "dl9": raw stresslet strengths (n, 9); "dl6": packed sym6
    (n, 6).  src_ids / trg_ids: fused exclusion (trg_ids per row of r_trg, -1 for targets that are not sources).
    select(rows, srcs) -> (R, C) multiplier of every pair (structure, defects)."""
    assert defect is None or defect in DEFECTS, defect
    r_src = np.asarray(r_src, dtype=np.float64).reshape(-1, 3)
    r_trg = np.asarray(r_trg, dtype=np.float64).reshape(-1, 3)
    rows = np.arange(r_trg.shape[0]) if rows is None else np.asarray(rows, dtype=np.int64)
    scale = scale_of(kind) if scale is None else LD(scale)
    if defect == "stresslet_sign":
        scale = -scale
    n = r_src.shape[0]
    block = max(n, 1) if block is None else block
    if kind == "sl":
        fs = np.asarray(f_src, dtype=np.float64).reshape(-1, 3).astype(LD)
        fa = np.abs(fs)
    else:
        fs, fa = _sym6(f_src, kind, defect)
    tid = None
    if src_ids is not None and trg_ids is not None:
        src_ids, tid = np.asarray(src_ids), np.asarray(trg_ids)[rows]
        if defect == "excl_by_position":
            run = int(np.argmax(src_ids != src_ids[0])) or n
            src_ids, tid = np.arange(n) // run, np.where(tid >= 0, rows // run, -1)
    t = r_trg[rows]
    nb = -(-n // block)
    ext = np.zeros((rows.size, nb, 3), dtype=LD)
    S = np.zeros((rows.size, nb, 3), dtype=LD)
    step = max(1, min(block, chunk // max(rows.size, 1)))
    for c in range(nb):
        for j0 in range(c * block, min(n, (c + 1) * block), step):
            srcs = np.arange(j0, min(n, (c + 1) * block, j0 + step))
            s = r_src[srcs]
            d64 = t[:, None, :] - s[None, :, :]                               # the kernels' rounded differences
            r2f = (d64 * d64).sum(axis=2)
            keep = r2f >= 4 * DBL_MIN                                         # far from the boundary either way
            near = ~keep
            if near.any():
                dn = d64[near]
                r2k = r2_kernel(dn[:, 0], dn[:, 1], dn[:, 2])
                keep[near] = r2k > 0 if defect == "no_subnormal_rule" else r2k >= DBL_MIN
            if tid is not None:
                keep &= tid[:, None] != src_ids[srcs][None, :]
            d = t[:, None, :].astype(LD) - s[None, :, :].astype(LD)
            term, aterm = _terms(kind, d, keep, fs[srcs][None], fa[srcs][None])
            if select is not None:
                m = np.asarray(select(rows, srcs), dtype=LD)[..., None]
                term, aterm = term * m, aterm * abs(m)
            ext[:, c] += term.sum(axis=1)
            S[:, c] += aterm.sum(axis=1)
    return ext * scale, S * abs(scale)


def pair_rows(*args, **kw):
    """(ext, S) of pair_blocks summed over the source runs: (len(rows), 3) each"""
    ext, S = pair_blocks(*args, **kw)
    return ext.sum(axis=1), S.sum(axis=1)


def combine(blocks, mult):
    """rows of a (R, nb, 3) block sum under a (R, nb) multiplier of the source runs"""
    return (blocks * np.asarray(mult, dtype=LD)[..., None]).sum(axis=1)


# ---- one pair in the kernels' float64 instruction order -------------------------------------------------------------
def seed(r2, eta):
    """a MUFU.RSQ64H stand-in: 1/sqrt(r2) (1 + eta) rounded to float64, eta within +-SEED_REL"""
    return ((1 / np.sqrt(np.asarray(r2, dtype=np.float64).astype(LD))) * (1 + LD(1) * eta)).astype(np.float64)


def _rsqrt(r2, eta, defect):
    y = np.where(r2 >= DBL_MIN, seed(np.where(r2 >= DBL_MIN, r2, 1.0), eta), 0.0)
    e = fma(-(r2 * y), y, 1.0)
    q = 0.5 * np.ones_like(e) if defect == "newton2" else fma(0.375, e, 0.5)
    return fma(y, e * q, y)


def pair_terms_f64(kind, t, s, f, eta, defect=None):
    """(N, 3) long-double terms the kernels add into their running sums for N pairs (t[k], s[k]) with strengths f[k]
    ((N, 3) packed Stokeslet, (N, 6) packed sym6 or (N, 9) raw stresslet): stokeslet_chains' y * v or
    stresslet_chains' d * co, every instruction in their order, the seed's relative error `eta`, the product exact
    (it is the fma of the accumulate)"""
    t, s = np.asarray(t, dtype=np.float64), np.asarray(s, dtype=np.float64)
    f = np.asarray(f, dtype=np.float64)
    dx, dy, dz = t[:, 0] - s[:, 0], t[:, 1] - s[:, 1], t[:, 2] - s[:, 2]
    r2 = r2_kernel(dx, dy, dz)
    y = _rsqrt(r2, eta, defect)
    if kind == "sl":
        fr = fma(f[:, 2], dz, fma(f[:, 1], dy, f[:, 0] * dx))
        q = fr * (y * y)
        v = np.stack([fma(dx, q, f[:, 0]), fma(dy, q, f[:, 1]), fma(dz, q, f[:, 2])], axis=1)
        return y.astype(LD)[:, None] * v.astype(LD)
    if kind == "dl9":
        off = (2 * f[:, 1], 2 * f[:, 2], 2 * f[:, 5]) if defect == "sym6_doubled" else \
            (f[:, 1] + f[:, 3], f[:, 2] + f[:, 6], f[:, 5] + f[:, 7])
        f = np.stack([f[:, 0], f[:, 4], f[:, 8], *off], axis=1)
    sxx, syy, szz, pxy, pxz, pyz = f.T
    co = fma(pxz, dz, fma(pxy, dy, sxx * dx))
    v2 = fma(pyz, dz, syy * dy)
    co = co * dx
    q = szz * dz
    co = fma(q, dz, fma(v2, dy, co))
    y2 = y * y
    co = co * ((y2 * y2) * y)
    d = np.stack([dx, dy, dz], axis=1)
    return d.astype(LD) * co.astype(LD)[:, None]


def accumulate(terms, order):
    """float64 running sums of (N, 3) long-double terms, each added by an fma (exact product, one rounding), visiting
    the terms in `order`"""
    u = np.zeros(3)
    for k in order:
        u = (terms[k] + u.astype(LD)).astype(np.float64)
    return u


# ---- rows to check ------------------------------------------------------------------------------------------------
def sample_rows(n_trg, periods=(), n_lead=None, ragged_period=None, n_random=256, seed=0, full_limit=2048):
    """sorted target rows: every row when n_trg <= full_limit; otherwise the first and last row of every tile of every
    period over [0, n_lead) (n_lead default n_trg), every row of the last, ragged tile of `ragged_period`, the remainder
    rows beyond n_lead (all of them when at most full_limit, else the edges of the plain kernel's tiles 128 T and their
    ragged last tiles) and n_random random rows"""
    if n_trg <= full_limit:
        return np.arange(n_trg)
    n_lead = n_trg if n_lead is None else n_lead
    out = [np.random.default_rng(seed).choice(n_trg, min(n_random, n_trg), replace=False)]

    def edges(lo, hi, ps, ragged):
        for p in ps:
            starts = np.arange(lo, hi, p)
            out.extend([starts, np.minimum(starts + p, hi) - 1])
        for p in ragged:
            last = lo + ((hi - lo - 1) // p) * p
            if hi > lo and hi - last < p:
                out.append(np.arange(last, hi))
    edges(0, n_lead, periods, [ragged_period] if ragged_period else [])
    if n_trg > n_lead:
        if n_trg - n_lead <= full_limit:
            out.append(np.arange(n_lead, n_trg))
        else:
            tiles = [CTA_THREADS * T for T in (1, 2, 4, 8)]
            edges(n_lead, n_trg, tiles, tiles)
    return np.unique(np.concatenate(out).astype(np.int64))

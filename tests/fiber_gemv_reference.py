"""Extended-precision restatement of the per-fiber GEMVs of fiber_gemv_kernel<MODE> (fiber_ops.cuh, launched from
FiberOps::force / matvec / precondition in skb_fiber.cu) -- TEST INFRASTRUCTURE ONLY.  Conventions of
tests/body_block_reference.py, whose U, ratio, _Ar, SLACK and k_gemv this module uses:

Every function takes float64 inputs and evaluates in `dtype`: np.longdouble gives `ext`, np.float64 a float64
restatement.  absolute=True gives the error scale S: every input by its absolute value, every subtraction an addition.
Sums run in the kernel's order: row r of a CTA is summed by 8 column slices (slice q takes columns q, q + 8, ... one
after the other; MODE 2's P terms c = rg.x + q, rg.x + q + 8, ... follow in the same accumulator and are subtracted
as one partial), then the 8 slice partials are added one after the other.  The float64 restatement therefore rounds as
the kernel does up to FMA contraction.

    fiber_force         MODE 1: force_operator_ x per fiber, scattered node-major (the apply_fiber_force layout)
    fiber_matvec        MODE 2: A_ x - P_downsample_bc vT(v) + xs_vT + y_BC (FiberFiniteDifference::matvec), with
                        vT = [v_x; v_y; v_z; D_1^T s], s_i = xs_i . v_i, D_1 = D_1_0 (2 / length_prev) applied as
                        the kernel does: the column sum over D_1_0's non-zero rows first, then one multiply by the
                        rounded 2 / length_prev.  P rows and D_1_0 columns are walked over the non-zero ranges
                        nonzero_ranges computes on the host: (0, 0) for a zero line, interior zeros spanned.
    fiber_precondition  MODE 0: A_^-1 x per fiber

A device value passes when |dev - ext| <= K u S entry by entry, u = 2^-53.  S of a P row carries the error that vT
itself carries: its terms are |P| [|v|; |D_1|^T (|xs| |v|)], not |P| |vT|.  Each K is the count of roundings on the
longest path from the float64 inputs to the entry (first order: an FMA counts one), plus SLACK, fixed from the code:

    MODE 0 / 1          k_gemv(4n): ceil(4n / 8) FMAs per slice, then the 7 slice additions.
    MODE 2              k_matvec(n, r_P, r_D) = k_gemv(4n)                        (the A_ x chain and the slice sums)
                          + ceil(r_P / 8)                                          (the P chain of a slice)
                          + 1                                                      (acc -= P partial)
                          + 3 + r_D + 2                                            (vT: s_i, the D_1_0 column chain,
                                                                                    2 / length_prev and the multiply)
                          + 3                                                      (the boundary row's additions:
                                                                                    xs_0 . v_0 or v_boundary, the
                                                                                    plus-end term)
                        r_P the longest non-zero range of a row of the fiber's P, r_D that of a column of its D_1_0.
                        Adding the A chain to the P path counts both in full: the bound is not tight, it is sound.

Planted defects (defect=), each a one-line slip the kernel or its host planning could make:

    drop_tail_column               a slice's last column of the j < cols tail loop is skipped (slices whose column
                                   count is not a multiple of 8 have a tail; MODE 0 / 1 / 2)
    drop_slice_7                   the last slice partial is left out of the row's sum (MODE 0 / 1 / 2)
    force_scatter_transposed       MODE 1 writes row k n + i to out[3 (off + k) + i] instead of out[3 (off + i) + k]
    d1_scale_inverted              D_1 = D_1_0 (length_prev / 2)
    p_range_short                  the P walk stops at rg.y - 1
    no_d_term_when_straddling_3n   a 32-row block whose P columns straddle column 3n gets no D_1^T s (its need_D
                                   tested as c_lo >= 3n); the block's vT[3n:] read as zero
    row3_missing_xs_v              boundary row 3 without xs_0 . v_0
    row10_ignores_plus_flag        boundary row 10 adds the last node's xs . v whether or not plus_velocity is set
    v_boundary_shifted             v_boundary[t] lands on boundary row t + 1
"""
import numpy as np

from body_block_reference import SLACK, U, _Ar, k_gemv, ratio  # noqa: F401  (U, ratio: for the tests)

ROWS = 32      # kFiberGemvRows
SLICES = 8     # kFiberGemvSlices
GEMV_DEFECTS = ("drop_tail_column", "drop_slice_7")
FORCE_DEFECTS = GEMV_DEFECTS + ("force_scatter_transposed",)
MATVEC_DEFECTS = GEMV_DEFECTS + ("d1_scale_inverted", "p_range_short", "no_d_term_when_straddling_3n",
                                 "row3_missing_xs_v", "row10_ignores_plus_flag", "v_boundary_shifted")
DEFECTS = FORCE_DEFECTS + MATVEC_DEFECTS[2:]


def nonzero_ranges(M, axis):
    """skb_fiber.cu nonzero_ranges: per row (axis=1) or column (axis=0) of M the first / one-past-last non-zero index,
    (0, 0) for a zero line.  Returns (lo, hi) int arrays."""
    nz = np.asarray(M) != 0.0
    if axis == 0:
        nz = nz.T
    any_ = nz.any(axis=1)
    lo = np.where(any_, nz.argmax(axis=1), 0)
    hi = np.where(any_, nz.shape[1] - nz[:, ::-1].argmax(axis=1), 0)
    return lo.astype(np.int64), hi.astype(np.int64)


def k_matvec(n, r_P, r_D):
    return k_gemv(4 * n) + int(np.ceil(r_P / SLICES)) + 1 + (3 + r_D + 2) + 3


def k_matvec_of(D_1_0, P):
    """k_matvec of one class from its matrices"""
    n = D_1_0.shape[0]
    lo, hi = nonzero_ranges(P, 1)
    dlo, dhi = nonzero_ranges(D_1_0, 0)
    return k_matvec(n, int((hi - lo).max(initial=0)), int((dhi - dlo).max(initial=0)))


def slice_partials(T, defect=None):
    """T (rows, cols) of terms in column order: per slice q the sum of columns q, q + 8, ... one after the other.
    Returns (8, rows).  drop_tail_column: a slice whose column count m_q has m_q mod 8 != 0 loses its last column."""
    rows, cols = T.shape
    m = -(-cols // SLICES) * SLICES
    P = np.zeros((rows, m), dtype=T.dtype)
    P[:, :cols] = T
    P = P.reshape(rows, m // SLICES, SLICES)           # [r, k, q]: column 8 k + q
    if defect == "drop_tail_column":
        for q in range(min(SLICES, cols)):
            m_q = (cols - q + SLICES - 1) // SLICES
            if m_q % 8:
                P[:, m_q - 1, q] = 0
    acc = P[:, 0, :].copy()
    for k in range(1, m // SLICES):
        acc = acc + P[:, k, :]
    return acc.T


def slice_sum(p, defect=None):
    """the row's sum of its 8 slice partials, added one after the other"""
    s = p[0]
    for u in range(1, SLICES - 1 if defect == "drop_slice_7" else SLICES):
        s = s + p[u]
    return s


def gemv(M, x, rows=None, dtype=np.longdouble, absolute=False, defect=None):
    """(M x)[rows] as fiber_gemv_kernel<0 / 1> sums it; rows None: all"""
    a = _Ar(dtype, absolute)
    rows = np.arange(M.shape[0]) if rows is None else np.asarray(rows)
    return slice_sum(slice_partials(a.v(M[rows]) * a.v(x)[None, :], defect), defect)


def fiber_force(F_list, x, n_nodes, dtype=np.longdouble, absolute=False, defect=None):
    """MODE 1 for every fiber: (N_f, 3), row k n + i of fiber f's force_operator_ x at [off_f + i, k]"""
    assert defect is None or defect in FORCE_DEFECTS, defect
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    out = np.zeros(3 * int(np.sum(n_nodes)), dtype=dtype)
    off = 0
    for F, n in zip(F_list, n_nodes):
        y = gemv(np.asarray(F), x[4 * off:4 * off + 4 * n], dtype=dtype, absolute=absolute,
                 defect=None if defect == "force_scatter_transposed" else defect)
        k, i = np.divmod(np.arange(3 * n), n)
        if defect == "force_scatter_transposed":
            out[3 * (off + k) + i] = y                 # (colliding writes: the last row wins)
        else:
            out[3 * (off + i) + k] = y
        off += n
    return out.reshape(-1, 3)


def fiber_precondition(Ainv_list, x, n_nodes, dtype=np.longdouble, absolute=False, defect=None):
    """MODE 0 for every fiber: A_^-1 x, (4 N_f,)"""
    assert defect is None or defect in GEMV_DEFECTS, defect
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    out, off = [], 0
    for M, n in zip(Ainv_list, n_nodes):
        out.append(gemv(np.asarray(M), x[4 * off:4 * off + 4 * n], dtype=dtype, absolute=absolute, defect=defect))
        off += n
    return np.concatenate(out) if out else np.zeros(0, dtype=dtype)


def _vT(a, D_1_0, xs, length_prev, v, defect):
    """[v_x; v_y; v_z; D_1^T s] as the kernel's preamble forms it"""
    n = xs.shape[0]
    vv, xt = a.v(v), a.v(xs)
    s = xt[:, 0] * vv[:, 0] + xt[:, 1] * vv[:, 1] + xt[:, 2] * vv[:, 2]
    D = a.v(D_1_0)
    acc = np.zeros(n, dtype=a.f)
    for i in range(n):                          # column j walks rows rg.x .. rg.y - 1; zero terms change nothing
        acc = acc + D[i, :] * s[i]
    lp, two = a.f(length_prev), a.f(2.0)
    scale = lp / two if defect == "d1_scale_inverted" else two / lp
    return np.concatenate([vv[:, 0], vv[:, 1], vv[:, 2], scale * acc])


def matvec_rows(A, D_1_0, P, xs, length_prev, plus, x, v, v_boundary=None, rows=None, dtype=np.longdouble,
                absolute=False, defect=None):
    """MODE 2 for one fiber, rows `rows` (None: all 4n) of A_ x - P vT + xs_vT + y_BC"""
    assert defect is None or defect in MATVEC_DEFECTS, defect
    a = _Ar(dtype, absolute)
    n = xs.shape[0]
    bc = 4 * n - 14
    rows = np.arange(4 * n) if rows is None else np.asarray(rows)
    gdef = defect if defect in GEMV_DEFECTS else None
    pa = slice_partials(a.v(A[rows]) * a.v(x)[None, :], gdef)            # (8, len(rows))
    vT = _vT(a, D_1_0, xs, length_prev, v, defect)
    prow = rows[rows < bc]
    if prow.size:
        lo, hi = nonzero_ranges(P[prow], 1)
        if defect == "p_range_short":
            hi = np.where(hi > lo, hi - 1, hi)
        vTr = np.broadcast_to(vT, (prow.size, 4 * n)).copy()
        if defect == "no_d_term_when_straddling_3n":
            # the CTA of each row: c_lo / c_hi over all its rows below bc
            glo, ghi = nonzero_ranges(P[:bc], 1)
            for j, r in enumerate(prow):
                r0 = r - r % ROWS
                blk = np.arange(r0, min(r0 + ROWS, bc))
                live = ghi[blk] > glo[blk]
                c_lo, c_hi = glo[blk][live].min(initial=4 * n), ghi[blk][live].max(initial=0)
                if c_lo < 3 * n < c_hi:
                    vTr[j, 3 * n:] = 0
        L = int((hi - lo).max(initial=0))
        idx = lo[:, None] + np.arange(L)[None, :]
        live = idx < hi[:, None]
        idx = np.where(live, idx, 0)
        terms = np.where(live, a.v(P[prow[:, None], idx]) * np.take_along_axis(vTr, idx, axis=1), a.f(0))
        pp = slice_partials(terms, None)
        sel = rows < bc
        pa[:, sel] = pa[:, sel] + a.sg * pp
    res = slice_sum(pa, gdef)
    vv, xt = a.v(v), a.v(xs)
    for j, r in enumerate(rows):
        t = int(r) - bc
        if t < 0:
            continue
        if t == 3 and defect != "row3_missing_xs_v":
            res[j] = res[j] + (vv[0, 0] * xt[0, 0] + vv[0, 1] * xt[0, 1] + vv[0, 2] * xt[0, 2])
        if v_boundary is not None:
            vb = a.v(v_boundary)
            tb = t - 1 if defect == "v_boundary_shifted" else t
            if 0 <= tb < 7:
                res[j] = res[j] + vb[tb]
        if t == 10 and (plus or defect == "row10_ignores_plus_flag"):
            e = n - 1
            res[j] = res[j] + (vv[e, 0] * xt[e, 0] + vv[e, 1] * xt[e, 1] + vv[e, 2] * xt[e, 2])
    return res


def fiber_matvec(ops, x, v, v_boundary=None, dtype=np.longdouble, absolute=False, defect=None):
    """MODE 2 for every fiber of `ops` (oracle.fiber_container_matvec's dict), (4 N_f,)"""
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    v = np.asarray(v, dtype=np.float64).reshape(-1, 3)
    out, off = [], 0
    for f, n in enumerate(ops["n_nodes"]):
        vb = None if v_boundary is None else np.asarray(v_boundary)[f]
        out.append(matvec_rows(ops["A"][f], ops["D_1_0"][n], ops["P"][n], ops["xs"][off:off + n],
                               ops["length_prev"][f], ops["plus"][f], x[4 * off:4 * off + 4 * n], v[off:off + n], vb,
                               dtype=dtype, absolute=absolute, defect=defect))
        off += n
    return np.concatenate(out) if out else np.zeros(0, dtype=dtype)


def k_rows(ops, mode):
    """K of every output entry of a container: mode 0 / 2 (4 N_f,), mode 1 (N_f, 3)"""
    out = []
    for n in ops["n_nodes"]:
        if mode == 2:
            out.append(np.full(4 * n, k_matvec_of(ops["D_1_0"][n], ops["P"][n]), dtype=np.float64))
        else:
            out.append(np.full(4 * n if mode == 0 else 3 * n, k_gemv(4 * n), dtype=np.float64))
    K = np.concatenate(out) if out else np.zeros(0)
    return K.reshape(-1, 3) if mode == 1 else K


def ext_and_scale(fn, *args, **kw):
    """(ext, S) of one of the functions above"""
    return fn(*args, dtype=np.longdouble, **kw), fn(*args, dtype=np.longdouble, absolute=True, **kw)

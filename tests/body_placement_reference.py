"""Extended-precision restatement of the placement of rigid bodies (body_place_kernel, skb_flow_place_bodies) -- TEST
INFRASTRUCTURE ONLY.  Conventions of tests/body_block_reference.py: float64 inputs evaluated in `dtype` (np.longdouble
gives `ext`, np.float64 a float64 restatement), absolute=True gives the error scale S.

R comes from the unit quaternion (w, x, y, z) by Eigen's toRotationMatrix formula (restated).  A placed inverse is
Y = Q X Q^T, Q = blockdiag(R, ..., R), tile by tile Y_IJ = R X_IJ R^T; a node's E_i = [ex_i ey_i ez_i] likewise.  The
kernel forms Z = X_IJ R^T, then R Z, each entry a three-term sum of products.

A device value passes when |dev - ext| <= K_PLACE u S entry by entry, S = S_R |X| S_R^T with S_R the formula of R on
absolute values (1 + |t_yy| + |t_zz| on the diagonal, |t_xy| + |t_wz| off it).  K_PLACE counts the roundings on the
longest path (first order): R from the quaternion, t_yy (1), t_yy + t_zz (1), 1 - that (1) = 3, entering twice (R and
R^T); Z, a three-term FMA chain or product sum (3); R Z, the same (3).  6 + 2 x 3 = 12, plus SLACK.
"""
import numpy as np

from body_block_reference import SLACK, U, ratio  # noqa: F401  (ratio: the callers' entry-wise measure)

K_PLACE = 12 + SLACK
DEFECTS = ("transpose", "static_motion_blocks", "previous_placement", "shift_tile")


def quaternion_rotation(q, dtype=np.longdouble, absolute=False):
    """R (3, 3) of the quaternion q = (w, x, y, z) (float64), or S_R with absolute=True"""
    w, x, y, z = (dtype(v) for v in np.asarray(q, dtype=np.float64))
    if absolute:
        w, x, y, z = abs(w), abs(x), abs(y), abs(z)
    sg = dtype(1) if absolute else dtype(-1)
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    one = dtype(1)
    return np.array([[one + sg * (tyy + tzz), txy + sg * twz, txz + twy],
                     [txy + twz, one + sg * (txx + tzz), tyz + sg * twx],
                     [txz + sg * twy, tyz + twx, one + sg * (txx + tyy)]], dtype=dtype)


def _rotate_tiles(T, Rl, Rr):
    """T[..., p, q] (3 x 3 tiles) -> Rl T Rr^T with the kernel's sums: Z = T Rr^T, then Rl Z, terms added in order"""
    Z = [T[..., :, 0] * Rr[b, 0] + T[..., :, 1] * Rr[b, 1] + T[..., :, 2] * Rr[b, 2] for b in range(3)]
    Z = np.stack(Z, axis=-1)                                          # Z[..., p, b]
    Y = [Rl[a, 0] * Z[..., 0, :] + Rl[a, 1] * Z[..., 1, :] + Rl[a, 2] * Z[..., 2, :] for a in range(3)]
    return np.stack(Y, axis=-2)                                       # Y[..., a, b]


def _R(q, dtype, absolute):
    return quaternion_rotation(q, dtype, absolute) if np.ndim(q) == 1 else np.asarray(q, dtype=dtype)


def place_column_tiles(X, q, tiles, dtype=np.longdouble, absolute=False):
    """columns [3J, 3J + 3) of Q X Q^T for the column tiles J in `tiles`: (m, 3 len(tiles))"""
    m = X.shape[0]
    cols = np.concatenate([np.arange(3 * J, 3 * J + 3) for J in tiles])
    Xc = np.asarray(X[:, cols], dtype=np.float64).astype(dtype)
    if absolute:
        Xc = np.abs(Xc)
    T = Xc.reshape(m // 3, 3, len(tiles), 3).transpose(0, 2, 1, 3)
    R = _R(q, dtype, absolute)
    return _rotate_tiles(T, R, R).transpose(0, 2, 1, 3).reshape(m, 3 * len(tiles))


def place_inverse(X, q, dtype=np.longdouble, absolute=False, defect=None, q_prev=None):
    """Q X Q^T of one body's (m, m) inverse (m = 3n + 6) at the quaternion q.  Defects: R^T in place of R; the two
    [U; w] tiles left unrotated; the rotation applied to the placement at q_prev instead of the frame; output tile
    (1, 0) taken from input tile (2, 0)."""
    assert defect is None or defect in DEFECTS, defect
    if defect == "previous_placement":
        X = place_inverse(X, q_prev, np.float64)
    R = _R(q, dtype, absolute)
    if defect == "transpose":
        R = R.T
    m = X.shape[0]
    k = m // 3
    Xf = np.asarray(X, dtype=np.float64).astype(dtype)
    if absolute:
        Xf = np.abs(Xf)
    T = Xf.reshape(k, 3, k, 3).transpose(0, 2, 1, 3)                  # T[I, J, p, q]
    if defect == "shift_tile":
        T = T.copy()
        T[1, 0] = T[2, 0]
    Y = _rotate_tiles(T, R, R)
    if defect == "static_motion_blocks":
        n = k - 2
        I3 = np.eye(3, dtype=dtype)
        Y[n:, :] = _rotate_tiles(T[n:, :], I3, R)
        Y[:, n:] = _rotate_tiles(T[:, n:], R, I3)
        Y[n:, n:] = T[n:, n:]
    return Y.transpose(0, 2, 1, 3).reshape(m, m)


def place_E(ex, ey, ez, q, dtype=np.longdouble, absolute=False, defect=None, q_prev=None):
    """R E_i R^T per node, E_i = [ex_i ey_i ez_i] (the (N, 3) arrays as columns); returns (ex, ey, ez).  Defects:
    transpose, previous_placement as in place_inverse."""
    assert defect in (None, "transpose", "previous_placement"), defect
    if defect == "previous_placement":
        ex, ey, ez = place_E(ex, ey, ez, q_prev, np.float64)
    R = _R(q, dtype, absolute)
    if defect == "transpose":
        R = R.T
    E = np.stack([np.asarray(a, dtype=np.float64) for a in (ex, ey, ez)], axis=-1).astype(dtype)  # E[i, p, c]
    if absolute:
        E = np.abs(E)
    Y = _rotate_tiles(E, R, R)
    return Y[:, :, 0], Y[:, :, 1], Y[:, :, 2]


def placed_geometry(pos_ref, nrm_ref, center, q):
    """the nodes and normals skb_flow_place_bodies forms on the host: c + R r, R n, sums in the same order (float64)"""
    R = quaternion_rotation(q, np.float64)
    r, n = np.asarray(pos_ref, dtype=np.float64), np.asarray(nrm_ref, dtype=np.float64)
    rot = lambda v: np.stack([R[k, 0] * v[:, 0] + R[k, 1] * v[:, 1] + R[k, 2] * v[:, 2] for k in range(3)], axis=1)
    return np.asarray(center, dtype=np.float64) + rot(r), rot(n)


def random_quaternions(rng, k):
    q = rng.normal(size=(k, 4))
    return q / np.linalg.norm(q, axis=1)[:, None]


def sphere_body(n, radius=0.5):
    """n Fibonacci nodes on a sphere about the origin, outward normals, equal quadrature weights 4 pi r^2 / n"""
    i = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * i / n)
    theta = np.pi * (1 + 5 ** 0.5) * i
    e = np.stack([np.cos(theta) * np.sin(phi), np.sin(theta) * np.sin(phi), np.cos(phi)], axis=1)
    return radius * e, e, np.full(n, 4 * np.pi * radius ** 2 / n)

"""CPU tests of the placement of rigid bodies (tests/body_placement_reference.py, which tests/test_gpu_body_placement.py
holds the device to): the identity A_(c, R) = Q A_0 Q^T and E_i(c, R) = R E_i,0 R^T on a real body, the entry-wise
criterion |dev - ext| <= K_PLACE u S attainable by a float64 evaluation, and every planted defect missing it."""
import numpy as np
import pytest

import body_placement_reference as bp
import system_reference as sr

DEFECT_FACTOR = 1e6  # the least factor (ratio / K) by which a defect must miss; each misses by far more


def test_rotation_is_eigens_formula_and_orthogonal():
    rng = np.random.default_rng(1)
    for q in bp.random_quaternions(rng, 20):
        R = bp.quaternion_rotation(q, np.float64)
        assert np.abs(R @ R.T - np.eye(3)).max() < 1e-15 and abs(np.linalg.det(R) - 1) < 1e-15
        v = rng.normal(size=3)  # R v = q v q* (the Hamilton product)
        w, u = q[0], q[1:]
        qv = v + 2 * w * np.cross(u, v) + 2 * np.cross(u, np.cross(u, v))
        assert np.allclose(R @ v, qv, rtol=0, atol=1e-14)
    assert np.array_equal(bp.quaternion_rotation([1.0, 0, 0, 0], np.float64), np.eye(3))


def test_identity_holds_on_a_real_body():
    """sphere nodes with quadrature weights: the operators evaluated at a placement equal the body-frame ones rotated"""
    r0, n0, w = bp.sphere_body(120)
    E0 = sr.singularity_vectors(r0, n0, w)
    A0 = sr.body_operator(r0, n0, np.zeros(3), w, *E0)
    rng = np.random.default_rng(2)
    q = bp.random_quaternions(rng, 1)[0]
    c = rng.uniform(-3, 3, 3)
    pos, nrm = bp.placed_geometry(r0, n0, c, q)
    E1 = sr.singularity_vectors(pos, nrm, w)
    A1 = sr.body_operator(pos, nrm, c, w, *E1)
    A_rot = bp.place_inverse(A0, q).astype(np.float64)
    assert np.abs(A_rot - A1).max() <= 1e-13 * np.abs(A1).max(), np.abs(A_rot - A1).max() / np.abs(A1).max()
    for got, ref in zip(bp.place_E(*E0, q), E1):
        assert np.abs(got.astype(np.float64) - ref).max() <= 1e-13 * np.abs(ref).max()
    # and so for the inverse: Q A_0^-1 Q^T inverts A_(c, R)
    Y = bp.place_inverse(np.linalg.inv(A0), q).astype(np.float64)
    x = rng.normal(size=A1.shape[0])
    res = np.linalg.norm(A1 @ (Y @ x) - x) / np.linalg.norm(x)
    res_host = np.linalg.norm(A1 @ np.linalg.solve(A1, x) - x) / np.linalg.norm(x)
    assert res <= max(10 * res_host, 1e-13), (res, res_host)
    print(f"\nreal body: |Q A_0 Q^T - A| / |A| = {np.abs(A_rot - A1).max() / np.abs(A1).max():.2e}; "
          f"inverse residual {res:.2e} (host solve {res_host:.2e})")


def _case(seed, n):
    rng = np.random.default_rng(seed)
    m = 3 * n + 6
    X = rng.normal(size=(m, m)) * 10.0 ** rng.uniform(-3, 3, m)[None, :]
    E = [rng.normal(size=(n, 3)) * 10.0 ** rng.uniform(-3, 3, (n, 1)) for _ in range(3)]
    return X, E, bp.random_quaternions(rng, 2)


@pytest.mark.parametrize("n", [1, 42, 400])
def test_float64_placement_meets_its_bound(n):
    X, E, (q, _) = _case(n, n)
    r = bp.ratio(bp.place_inverse(X, q, np.float64), bp.place_inverse(X, q), bp.place_inverse(X, q, absolute=True))
    ext, S = bp.place_E(*E, q), bp.place_E(*E, q, absolute=True)
    rE = max(bp.ratio(g, e, s).max() for g, e, s in zip(bp.place_E(*E, q, np.float64), ext, S))
    assert r.max() <= bp.K_PLACE and rE <= bp.K_PLACE, (r.max(), rE)
    print(f"\nfloat64 placement, n = {n}: inverse {r.max():.2f}, E {rE:.2f} (K {bp.K_PLACE})")


@pytest.mark.parametrize("defect", bp.DEFECTS)
def test_criterion_catches_planted_defects(defect):
    X, E, (q, q_prev) = _case(5, 42)
    ext, S = bp.place_inverse(X, q), bp.place_inverse(X, q, absolute=True)
    bad = bp.place_inverse(X, q, np.float64, defect=defect, q_prev=q_prev)
    f = bp.ratio(bad, ext, S).max() / bp.K_PLACE
    if defect in ("transpose", "previous_placement"):
        extE, SE = bp.place_E(*E, q), bp.place_E(*E, q, absolute=True)
        badE = bp.place_E(*E, q, np.float64, defect=defect, q_prev=q_prev)
        f = min(f, max(bp.ratio(g, e, s).max() for g, e, s in zip(badE, extE, SE)) / bp.K_PLACE)
    print(f"\n{defect}: misses its bound by {f:.3g} x K")
    assert f > DEFECT_FACTOR, (defect, f)

"""CPU tests of the periphery restatement (tests/periphery_reference.py) against hand-derived cases: the repulsion in a
sphere and an ellipsoid, the binding window, the clamped node 0 and the body collisions."""
import numpy as np
import pytest

import periphery_reference as pr

SPHERE = dict(kind="sphere", a=5.0, b=0.0, c=0.0, f_0=20.0, l_0=0.5, binding_active=True, polar_angle_start=0.0,
              polar_angle_end=np.pi / 2, binding_threshold=0.75)
ELLIPSOID = dict(SPHERE, kind="ellipsoid", a=7.8, b=4.16, c=4.16)


@pytest.mark.parametrize("dtype", [np.float64, np.longdouble])
def test_radial_nodes_in_a_sphere(dtype):
    rng = np.random.default_rng(1)
    u = rng.normal(size=(20, 3))
    u /= np.linalg.norm(u, axis=1)[:, None]
    r = rng.uniform(0.1, 4.9, 20)
    f = pr.fiber_interaction(SPHERE, u * r[:, None], dtype=dtype)
    want = -20.0 * u * np.exp(-(5.0 - r) / 0.5)[:, None]  # the force points to the centre: -f_0 u exp(-(R - r)/l_0)
    np.testing.assert_allclose(np.asarray(f, dtype=np.float64), want, rtol=1e-12, atol=0)


@pytest.mark.parametrize("shape", [SPHERE, ELLIPSOID], ids=["sphere", "ellipsoid"])
def test_nodes_on_or_outside_the_surface_get_zero(shape):
    x = np.array([[shape["a"], 0.0, 0.0], [0.0, 0.0, 9.0], [10.0, 10.0, 10.0], [0.0, -8.0, 0.0]])
    assert not pr.fiber_interaction(shape, x).any()
    assert pr.outside(shape, x).all()


def test_ellipsoid_axis_points():
    # on the x axis the cortex point is (a, 0, 0): dr = (x - a, 0, 0), the force -f_0 x_hat exp(-(a - x)/l_0)
    x = np.array([[3.0, 0.0, 0.0], [-2.0, 0.0, 0.0]])
    f = pr.fiber_interaction(ELLIPSOID, x)
    # (c cos(theta) rounds to ~1e-19, not 0)
    np.testing.assert_allclose(f[0], [-20.0 * np.exp(-(7.8 - 3.0) / 0.5), 0, 0], rtol=1e-9, atol=1e-15)
    # on the z axis the cortex lies near (0, 0, c): the 1e-12 guard in acos tilts theta by ~sqrt(2e-12) from 0, so
    # the force has a small x component, as in the reference
    z = pr.fiber_interaction(ELLIPSOID, np.array([[0.0, 0.0, 4.0]]))
    np.testing.assert_allclose(z[0, 2], -20.0 * np.exp(-(4.16 - 4.0) / 0.5), rtol=1e-8)
    assert z[0, 1] == 0 and 0 < -z[0, 0] < 1e-2
    assert f[1, 0] > 0


def test_polar_angle_window_and_zero_last_node():
    near = np.array([[0.0, 0.0, 1.0], [0.0, 0.0, 4.5]])  # within 0.75 of the sphere, last node at angle 0
    assert pr.plus_hinged(SPHERE, near)
    below = near * np.array([1, 1, -1])  # angle pi: outside [0, pi/2]
    assert not pr.plus_hinged(SPHERE, below)
    zero_last = np.array([[4.6, 0.0, 0.0], [0.0, 0.0, 0.0]])  # normalized(0) = 0: angle pi/2, inside the window
    assert pr.polar_angle(zero_last[-1]) == np.pi / 2
    assert pr.plus_hinged(SPHERE, zero_last)
    assert not pr.plus_hinged(dict(SPHERE, polar_angle_end=1.5), zero_last)
    assert not pr.plus_hinged(dict(SPHERE, binding_active=False), near)
    far = np.array([[0.0, 0.0, 1.0], [0.0, 0.0, 2.0]])
    assert not pr.plus_hinged(SPHERE, far)


def test_minus_clamped_against_body_bound():
    # node 0 beyond the surface: the force skips it only on the TOML flag, the collision test on is_minus_clamped()
    x = np.array([[6.0, 0.0, 0.0], [4.0, 0.0, 0.0], [3.0, 0.0, 0.0]])
    toml = pr.fiber_interaction(SPHERE, x, minus_clamped=True)
    bound = pr.fiber_interaction(SPHERE, x, minus_clamped=False)
    assert not toml[0].any() and not bound[0].any()  # node 0 is outside: no force either way
    inside0 = np.array([[2.0, 0.0, 0.0], [4.0, 0.0, 0.0]])
    assert not pr.fiber_interaction(SPHERE, inside0, minus_clamped=True)[0].any()
    assert pr.fiber_interaction(SPHERE, inside0, minus_clamped=False)[0, 0] < 0
    # a body-bound fiber (is_minus_clamped, not minus_clamped_) skips node 0 in the collision test only
    assert not pr.fibers_collided(SPHERE, [x], [True])
    assert pr.fibers_collided(SPHERE, [x], [False])


def test_touching_and_separated_bodies():
    c = np.array([[0.0, 0.0, 0.0], [2.0, 0.0, 0.0]])
    assert not pr.bodies_collided(SPHERE, c, [1.0, 1.0])  # touching: |c1 - c2|^2 = (r1 + r2)^2 is not <
    assert pr.bodies_collided(SPHERE, c, [1.0, 1.0 + 1e-9])
    assert not pr.bodies_collided(SPHERE, c, [1.0, 0.0])  # not spherical: never colliding
    assert pr.bodies_collided(SPHERE, [[4.5, 0.0, 0.0]], [0.6])  # |c| + r > R
    assert not pr.bodies_collided(ELLIPSOID, [[7.5, 0.0, 0.0]], [0.6])  # the ellipsoid's stub: false
    assert pr.check_collision(SPHERE, [np.zeros((2, 3))], [False], c, [1.5, 1.0])

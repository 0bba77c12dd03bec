"""Restatement of SphericalPeriphery / EllipsoidalPeriphery::fiber_interaction (periphery.cpp:140-162, 232-263),
::check_collision (periphery.cpp:94-97, 126-133, 204-224), FiberFiniteDifference::update_boundary_conditions
(fiber_finite_difference.cpp:74-91), FiberContainerFiniteDifference::check_collision (fcfd.cpp:39-54) and
SphericalBody::check_collision (body_spherical.cpp:304-307) in numpy, in float64 or np.longdouble (dtype=...).

A shape is a dict: kind ("sphere" / "ellipsoid"), a, b, c, f_0, l_0, binding_active, polar_angle_start,
polar_angle_end, binding_threshold."""
import numpy as np


def _cortex(shape, x, t, dt):
    """the point of the ellipsoid with semi-axes shrunk by t in the direction of each row of x, the reference's 1e-12
    guards in atan2 and acos"""
    abc = np.array([shape["a"], shape["b"], shape["c"]], dtype=dt)
    rs = x / abc
    rs_mag = np.sqrt(np.sum(rs * rs, axis=1))
    eps = dt(1e-12)
    phi = np.arctan2(rs[:, 1], rs[:, 0] + eps)
    theta = np.arccos(rs[:, 2] / (eps + rs_mag))
    st = np.sin(theta)
    t = dt(t)
    return np.stack([(abc[0] - t) * st * np.cos(phi), (abc[1] - t) * st * np.sin(phi), (abc[2] - t) * np.cos(theta)],
                    axis=1)


def outside(shape, x, threshold=0.0, dtype=np.float64):
    """Periphery::check_collision per point (rows of x): on or beyond the surface shrunk by threshold"""
    x = np.asarray(x, dtype=dtype).reshape(-1, 3)
    r2 = np.sum(x * x, axis=1)
    if shape["kind"] == "sphere":
        R = dtype(shape["a"]) - dtype(threshold)
        return r2 >= R * R
    rc = _cortex(shape, x, threshold, dtype)
    return r2 >= np.sum(rc * rc, axis=1)


def fiber_interaction(shape, x, minus_clamped=False, dtype=np.float64):
    """the repulsion (n, 3) on the nodes x (n, 3) of one fiber; node 0 skipped when minus_clamped (the TOML flag)"""
    x = np.asarray(x, dtype=dtype).reshape(-1, 3)
    f = np.zeros_like(x)
    r_mag = np.sqrt(np.sum(x * x, axis=1))
    if shape["kind"] == "sphere":
        R = np.full(len(x), dtype(shape["a"]))
        with np.errstate(invalid="ignore", divide="ignore"):
            surf = x / r_mag[:, None] * R[:, None]
    else:
        surf = _cortex(shape, x, 0.0, dtype)
        R = np.sqrt(np.sum(surf * surf, axis=1))
    inside = r_mag < R
    inside[:1] &= not minus_clamped
    dr = x - surf
    d = np.sqrt(np.sum(dr * dr, axis=1))
    with np.errstate(invalid="ignore", divide="ignore"):
        val = dtype(shape["f_0"]) * dr / d[:, None] * np.exp(-(R - r_mag) / dtype(shape["l_0"]))[:, None]
    f[inside] = val[inside]
    return f


def polar_angle(x_last, dtype=np.float64):
    """acos(x_last.normalized()[2]); Eigen's normalized() of a zero vector is the zero vector"""
    q = np.asarray(x_last, dtype=dtype)
    z2 = np.sum(q * q)
    return np.arccos(q[2] / np.sqrt(z2) if z2 > 0 else dtype(0))


def plus_hinged(shape, x, dtype=np.float64):
    """update_boundary_conditions' bc_plus_ hinge of one fiber"""
    x = np.asarray(x, dtype=dtype).reshape(-1, 3)
    if not shape["binding_active"]:
        return False
    ang = polar_angle(x[-1], dtype)
    return bool(shape["polar_angle_start"] <= ang <= shape["polar_angle_end"]
                and outside(shape, x, shape["binding_threshold"], dtype).any())


def fibers_collided(shape, fibers, is_minus_clamped, dtype=np.float64):
    """FiberContainerFiniteDifference::check_collision at threshold 0: node 0 skipped when is_minus_clamped"""
    return any(outside(shape, np.asarray(x)[1 if c else 0:], 0.0, dtype).any() for x, c in zip(fibers, is_minus_clamped))


def bodies_collided(shape, centers, radius, dtype=np.float64):
    """spherical bodies (radius > 0) against a spherical periphery and against each other, threshold 0"""
    c = np.asarray(centers, dtype=dtype).reshape(-1, 3)
    r = np.asarray(radius, dtype=dtype)
    for i in range(len(c)):
        if r[i] <= 0:
            continue
        if shape["kind"] == "sphere" and np.sqrt(np.sum(c[i] * c[i])) + r[i] > dtype(shape["a"]):
            return True
        for j in range(len(c)):
            if j != i and r[j] > 0 and np.sum((c[i] - c[j]) ** 2) < (r[i] + r[j]) ** 2:
                return True
    return False


def check_collision(shape, fibers, is_minus_clamped, centers=(), radius=(), dtype=np.float64):
    """System::check_collision: any fiber or body collision"""
    return fibers_collided(shape, fibers, is_minus_clamped, dtype) or bodies_collided(shape, centers, radius, dtype)

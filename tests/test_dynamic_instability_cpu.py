"""CPU tests of tests/dynamic_instability_reference.py, the restatement skb_flow_dynamic_instability is held to bitwise:
the Philox4x32-10 known answers, the model's cases and the laws of its draws."""
import math

import numpy as np
import pytest

import dynamic_instability_reference as dr
from skellysim_b200.capi import FIBER_PARAMS_DTYPE


@pytest.mark.parametrize("ctr, key, want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    assert dr.philox4x32_10(ctr, key) == want


def test_uniform_is_in_the_unit_interval_and_uses_53_bits():
    u = [dr.uniform(7, 3, i, dr.CATASTROPHE) for i in range(1000)]
    assert all(0.0 <= v < 1.0 for v in u)
    assert all(v * 2.0 ** 53 == int(v * 2.0 ** 53) for v in u)
    assert dr.uniform(7, 3, 0, 0) != dr.uniform(7, 3, 0, 1) != dr.uniform(7, 4, 0, 1)


DI = dict(n_nodes=16, v_growth=0.5, f_catastrophe=2.0, v_grow_collision_scale=0.25, f_catastrophe_collision_scale=4.0,
          nucleation_rate=3.0, radius=0.0125, min_length=0.3, bending_rigidity=2.5e-3)


def system(n_fibers=40, sites=(30, 20), seed=3):
    rng = np.random.default_rng(seed)
    params = np.zeros(n_fibers, dtype=FIBER_PARAMS_DTYPE)
    params["length_prev"], params["bending_rigidity"], params["radius"] = 0.9, 2.5e-3, 0.0125
    params["penalty_param"], params["beta_tstep"] = 500.0, 1.0
    lengths = rng.uniform(0.5, 1.5, n_fibers)
    binding = np.full((n_fibers, 2), -1)
    off = np.concatenate([[0], np.cumsum(sites)])
    flat = rng.permutation(int(off[-1]))[:n_fibers // 2]
    for f, s in enumerate(flat):
        b = int(np.searchsorted(off, s, side="right") - 1)
        binding[f] = (b, s - off[b])
    pinned = (rng.uniform(size=n_fibers) < 0.3).astype(int)
    site_ref = rng.normal(size=(int(off[-1]), 3))
    centers = rng.normal(size=(len(sites), 3))
    q = rng.normal(size=(len(sites), 4))
    q /= np.linalg.norm(q, axis=1)[:, None]
    return dict(lengths=lengths, params=params, binding=binding, plus_pinned=pinned, sites_per_body=list(sites),
                site_ref=site_ref, centers=centers, quats=q)


def call(di, sysd, dt=0.05, seed=11, counter=0):
    return dr.dynamic_instability(di, dt, seed, counter, **sysd)


def test_n_nodes_zero_is_the_identity():
    s = system()
    out = call(dict(DI, n_nodes=0), s)
    assert np.array_equal(out["lengths"], s["lengths"]) and np.array_equal(out["params"], s["params"])
    assert np.array_equal(out["origin"], np.arange(40)) and out["removed"] == out["nucleated"] == 0


def test_no_catastrophe_and_no_nucleation_is_growth_only():
    s = system()
    out = call(dict(DI, f_catastrophe=0.0, nucleation_rate=0.0), s)
    v = np.where(s["plus_pinned"] == 1, 0.5 * 0.25, 0.5)
    assert out["removed"] == 0 and out["nucleated"] == 0 and out["mu"] == 0.0
    assert np.array_equal(out["lengths"], s["lengths"] + 0.05 * v)
    assert np.array_equal(out["params"]["length_prev"], s["lengths"])
    assert np.array_equal(out["v_growth"], v) and np.array_equal(out["binding"], s["binding"])


def test_the_pinned_scales_apply():
    s = system()
    s["plus_pinned"][:] = 1
    out = call(dict(DI, f_catastrophe_collision_scale=0.0, nucleation_rate=0.0), s)
    assert out["removed"] == 0 and np.all(out["v_growth"] == 0.5 * 0.25)
    s["plus_pinned"][:] = 0
    out = call(dict(DI, f_catastrophe=1e6, f_catastrophe_collision_scale=0.0, nucleation_rate=0.0), s)
    assert out["removed"] == 40


def test_the_count_is_capped_by_the_free_sites_and_new_fibers_are_straight():
    s = system(n_fibers=10, sites=(6, 4))
    out = call(dict(DI, f_catastrophe=0.0, nucleation_rate=1e6), s)
    bound = int((s["binding"][:, 0] >= 0).sum())
    assert out["nucleated"] == 10 - bound and out["mu"] > 1e4
    flat = [int(np.sum([6, 4][:b])) + st for b, st in out["binding"] if b >= 0]
    assert len(set(flat)) == len(flat) == 10  # every site once
    x = dr.straight_fiber(s["centers"][0], s["quats"][0], s["site_ref"][0], 16, 0.3)
    seg = np.linalg.norm(np.diff(x, axis=0), axis=1)
    assert np.allclose(seg, 0.3 / 15, rtol=1e-12) and x.shape == (16, 3)
    assert np.all(out["params"]["minus_clamped"][-out["nucleated"]:] == 1)
    assert np.all(out["params"]["plus_hinged"][-out["nucleated"]:] == 0)


def test_all_fibers_die():
    s = system()
    out = call(dict(DI, f_catastrophe=1e6, f_catastrophe_collision_scale=1.0, nucleation_rate=0.0), s)
    assert out["removed"] == 40 and len(out["origin"]) == 0 and out["lengths"].size == 0


@pytest.mark.parametrize("sites", [(), (0, 0)])
def test_no_bodies_or_no_sites(sites):
    s = system(sites=sites)
    s["binding"][:] = -1
    out = call(dict(DI, nucleation_rate=5.0), s)
    assert out["nucleated"] == 0 and out["mu"] == 0.0 and out["grown"] + out["removed"] == 40


@pytest.mark.parametrize("mu", [0.3, 30.0, 3000.0])
def test_poisson_mean_and_variance(mu):
    n = 100_000
    k = np.array([dr.poisson(mu, 5, c) for c in range(n)], dtype=np.float64)
    se_mean = math.sqrt(mu / n)
    se_var = mu * math.sqrt((2.0 + 1.0 / mu) / n)  # var of the sample variance of a Poisson: (mu + 2 mu^2) / n
    assert abs(k.mean() - mu) <= 5 * se_mean, (k.mean(), mu)
    assert abs(k.var() - mu) <= 5 * se_var, (k.var(), mu)


def test_poisson_of_zero_mean_is_zero():
    assert dr.poisson(0.0, 5, 0) == 0


def test_catastrophe_fraction():
    n, dt, f = 20_000, 0.05, 3.0
    s = system(n_fibers=n, sites=())
    s["binding"][:] = -1
    s["plus_pinned"][:] = 0
    out = call(dict(DI, f_catastrophe=f, nucleation_rate=0.0), s, dt=dt)
    p = 1 - math.exp(-dt * f)
    assert abs(out["removed"] / n - p) <= 5 * math.sqrt(p * (1 - p) / n)

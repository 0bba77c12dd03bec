"""CPU tests of tests/step_reference.py against the reference's own statements (System::step, fiber_error_local,
System::run), of the planted defects it must catch, and of skellysim_b200.timestep.run on a scripted stepper."""
import numpy as np
import pytest

import step_reference as st
from oracle.fiber_fd import compute_matrices
from skellysim_b200 import timestep

U = 2.0 ** -53


def straight(n, L, scale=1.0, seed=0):
    rng = np.random.default_rng(seed)
    t = rng.normal(size=3)
    t /= np.linalg.norm(t)
    return rng.normal(size=3) + np.linspace(0.0, scale * L, n)[:, None] * t


def rodrigues(phi):
    a = np.linalg.norm(phi)
    k = phi / a
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(a) * K + (1 - np.cos(a)) * K @ K


@pytest.mark.parametrize("n", [8, 32, 128])
def test_straight_fiber_error_is_rounding_and_a_stretch_is_its_strain(n):
    D = compute_matrices(n)["D_1_0"]
    L = 1.7
    e, S = st.fiber_error(straight(n, L), L, D)
    assert e.max() <= 64 * U * S.max(), e.max()
    for eps in (1e-3, 1e-6):
        e, _ = st.fiber_error(straight(n, L, 1 + eps), L, D)
        assert e.max() == pytest.approx(eps, rel=1e-6)
    e_ld, _ = st.fiber_error(straight(n, L, 1 + 1e-3), L, D, dtype=np.longdouble)
    assert float(e_ld.max()) == pytest.approx(1e-3, rel=1e-9)


def test_planted_fiber_error_defects_miss_by_a_wide_margin():
    n, L = 32, 1.3
    D = compute_matrices(n)["D_1_0"]
    pos = straight(n, L)
    good = st.fiber_error(pos, L, D)[0].max()
    assert good < 1e-12
    assert st.fiber_error(pos, 0.8 * L, D)[0].max() > 0.1      # length_prev (here 0.8 L) in place of length_
    assert st.fiber_error(pos, L, D, scale=1.0)[0].max() > 0.4  # 1/L in place of 2/L


def test_q_new_is_the_rotation_by_phi_composed_on_the_left_and_q_phi_on_the_right_is_caught():
    rng = np.random.default_rng(1)
    for _ in range(50):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        w, dt = rng.normal(size=3), 0.3
        c_new, q_new = st.body_step(np.zeros(3), q, np.zeros(3), w, dt)
        want = rodrigues(w * dt) @ st.rotation(q)
        assert np.abs(st.rotation(q_new) - want).max() <= 1e-14
        _, q_bad = st.body_step(np.zeros(3), q, np.zeros(3), w, dt, right=True)
        assert np.abs(st.rotation(q_bad) - want).max() > 1e-3


def test_a_million_body_steps_keep_q_unit():
    rng = np.random.default_rng(2)
    m, steps, dt = 1000, 1000, 0.05
    q = rng.normal(size=(m, 4))
    q /= np.linalg.norm(q, axis=1)[:, None]
    for _ in range(steps):  # body_step vectorised over m bodies, in its operation order
        w = rng.normal(size=(m, 3))
        phi = w * dt
        pn = np.sqrt(phi[:, 0] * phi[:, 0] + phi[:, 1] * phi[:, 1] + phi[:, 2] * phi[:, 2])
        sh = np.sin(0.5 * pn)
        qp = np.stack([np.cos(0.5 * pn), sh * phi[:, 0] / pn, sh * phi[:, 1] / pn, sh * phi[:, 2] / pn])
        r = st.quat_mul(qp, q.T).T
        q = r / np.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])[:, None]
    drift = np.abs((q * q).sum(axis=1) - 1.0).max()
    assert drift <= 1e-13, drift
    # one body through body_step itself agrees with the vectorised form's rule
    c, q1 = st.body_step(np.zeros(3), q[0], np.ones(3), np.array([0.1, 0.2, 0.3]), dt)
    assert abs((q1 * q1).sum() - 1) <= 4 * U and np.array_equal(c, np.full(3, dt))


def test_the_literal_rule_translates_only_when_it_turns():
    c, q = np.array([1.0, 2.0, 3.0]), np.array([1.0, 0, 0, 0])
    U_, dt = np.array([0.5, 0.0, -1.0]), 0.1
    assert np.array_equal(st.body_step(c, q, U_, np.zeros(3), dt, literal=True)[0], c)
    assert np.array_equal(st.body_step(c, q, U_, np.zeros(3), dt)[0], c + U_ * dt)
    w = np.array([0.0, 0.3, 0.0])
    assert np.array_equal(st.body_step(c, q, U_, w, dt, literal=True)[0], st.body_step(c, q, U_, w, dt)[0])


def test_repin_puts_node_0_on_the_site_and_the_planted_defects_miss():
    rng = np.random.default_rng(3)
    for _ in range(100):
        pos = rng.normal(size=(16, 3)) * 10
        s = rng.normal(size=3) * 10
        r = st.repin(pos, s)
        assert np.all(np.abs(r[0] - s) <= 2 * U * (np.abs(pos[0]) + np.abs(s)))
        assert np.allclose(np.diff(r, axis=0), np.diff(pos, axis=0), rtol=0, atol=1e-13)
        assert np.abs(st.repin(pos, s, from_last=True)[0] - s).max() > 1e-3
    c, q = np.array([1.0, 0, 0]), np.array([np.cos(0.4), np.sin(0.4), 0, 0])
    s_ref = np.array([0.0, 0.5, 0.0])
    assert np.linalg.norm(st.site(c, q, s_ref) - st.site(c, q, s_ref, rotate=False)) > 0.1


def test_fiber_step_deinterleaves_the_solution_block():
    n_nodes = [4, 6]
    x = np.arange(4 * sum(n_nodes), dtype=float)
    (p0, t0), (p1, t1) = st.fiber_step(x, n_nodes)
    assert np.array_equal(p0[:, 1], x[4:8]) and np.array_equal(t0, x[12:16])
    assert np.array_equal(p1[2], x[16 + np.array([2, 8, 14])]) and np.array_equal(t1, x[34:40])


# ---- the run loop on a scripted stepper ------------------------------------------------------------------------------


class ScriptedStepper:
    """(converged, fiber_error, collided) per step; positions change on every step and restore undoes them"""

    def __init__(self, outcomes):
        self.outcomes, self.k, self.state, self.restores, self.dts = list(outcomes), 0, 0, [], []
        self._collided = False

    def positions(self):
        return np.full((1, 3), float(self.state))

    def placement(self):
        return np.zeros((0, 3)), np.zeros((0, 4))

    def backup(self):
        self.saved = self.state

    def restore(self):
        self.restores.append(self.k - 1)
        self.state = self.saved

    def step(self, dt, f_external=None, body_forces_torques=None):
        converged, err, self._collided = self.outcomes[self.k]
        self.k += 1
        self.state += 1
        self.dts.append(dt)
        return dict(converged=int(converged), fiber_error=err)

    def collided(self, r, c):
        return self._collided


KW = dict(dt_min=1e-4, dt_max=0.1, beta_up=1.2, beta_down=0.5, fiber_error_tol=0.1)


def drive(outcomes, dt=0.01, t_final=0.05, adaptive=True, **over):
    kw = dict(KW, **over)
    s = ScriptedStepper(outcomes)
    t, dt_end, log = timestep.run(s, t_final, dt, adaptive=adaptive, collided=s.collided, **kw)
    ref = st.run_reference(outcomes, dt, t_final, kw["dt_min"], kw["dt_max"], kw["beta_up"], kw["beta_down"],
                           kw["fiber_error_tol"], adaptive=adaptive)
    return s, t, log, ref


def test_run_follows_the_references_decisions_and_restores_exactly_on_rejects():
    rng = np.random.default_rng(4)
    outcomes = [(rng.uniform() > 0.05, rng.uniform(0, 0.105), rng.uniform() > 0.97) for _ in range(2000)]
    s, t, log, ref = drive(outcomes, t_final=0.3, dt_min=1e-300)
    assert [(a, b, c) for a, b, c, _ in log] == ref
    assert s.restores == [k for k, (_, _, acc) in enumerate(ref) if not acc]
    assert t == ref[-1][0] >= 0.3 and len(set(s.dts)) > 10
    assert s.state == sum(acc for _, _, acc in ref)


def test_run_grows_dt_to_dt_max_and_ends_at_t_final():
    s, t, log, ref = drive([(True, 0.0, False)] * 200, dt=0.01, t_final=1.0)
    assert not s.restores and max(s.dts) == KW["dt_max"]
    assert t >= 1.0 and t - log[-1][1] < 1.0


def test_run_raises_below_dt_min_and_accepts_everything_without_adaptivity():
    with pytest.raises(RuntimeError, match="dt_min"):
        drive([(False, 0.0, False)] * 50)
    s, t, log, ref = drive([(False, 9.0, True)] * 10, adaptive=False)
    assert not s.restores and all(a for _, _, a, _ in log) and len(log) == 5


def test_time_advanced_by_the_grown_dt_is_caught():
    outcomes = [(True, 0.0, False)] * 20
    ours = st.run_reference(outcomes, 0.01, 0.05, 1e-4, 0.1, 1.2, 0.5, 0.1)
    literal = st.run_reference(outcomes, 0.01, 0.05, 1e-4, 0.1, 1.2, 0.5, 0.1, literal=True)
    s, t, log, _ = drive(outcomes)
    assert [r[0] for r in ours] == [l[0] for l in log]
    assert abs(literal[0][0] - log[0][0]) >= 0.0019  # the first step alone: 0.012 instead of 0.01

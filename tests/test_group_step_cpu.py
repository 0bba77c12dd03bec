"""CPU tests of distributed.RankStepper's bookkeeping (no GPU): it hands a group member's step the own fibers' slices of
the per-fiber arguments and of f_external, over the partitions of skb_mflow (capi.partition_query), and those slices
tile the complete arrays."""
import ctypes as C

import numpy as np
import pytest

from skellysim_b200 import capi, distributed


class RecordingFlow:
    """what RankStepper reads of a capi.Flow, and a group_step_device that records what it was given"""

    def __init__(self, fiber_n, n_shell, body_n, partition):
        self._fiber_off = np.concatenate([[0], np.cumsum(fiber_n)]).astype(np.int64)
        self._lengths = np.linspace(0.5, 1.0, len(fiber_n))
        self.n_fib, self.n_shell, self._body_n, self.n_bodies = int(self._fiber_off[-1]), n_shell, body_n, len(body_n)
        self._ranges = partition
        self.calls = []

    def group_step_device(self, *params, **kw):
        a, b = (int(self._fiber_off[v]) for v in self._ranges[:2])
        read = lambda ptr, n: (np.ctypeslib.as_array((C.c_double * n).from_address(ptr)).copy() if ptr else None)
        rec = dict(kw, params=params)
        rec["f_external"] = read(kw["d_f_external"], 3 * (b - a))
        rec["forces"] = read(kw["d_body_forces"], 3 * self.n_bodies)
        rec["torques"] = read(kw["d_body_torques"], 3 * self.n_bodies)
        self.calls.append(rec)
        return dict(converged=1, fiber_error=0.0, worst_fiber=-1)


def fibers(seed):
    rng = np.random.default_rng(seed)
    n = rng.integers(8, 20, size=7)
    return n, int(n.sum())


@pytest.mark.parametrize("world", [2, 3])
def test_rank_stepper_slices_to_the_own_fibers_and_the_slices_tile(world):
    fiber_n, n_fib = fibers(world)
    nfib, n_shell, body_n = len(fiber_n), 30, [12, 9]
    rng = np.random.default_rng(5)
    lengths = rng.uniform(0.5, 1.0, nfib)
    params = (lengths, rng.uniform(1e-3, 1e-2, nfib), 0.0125, 500.0, 1.0, np.arange(nfib) % 2, 0)
    fiber_body = np.array([0, 1, -1, 0, -1, 1, -1])
    site_ref = rng.normal(size=(nfib, 3))
    v_growth, force_scale = rng.normal(size=nfib), rng.normal(size=nfib)
    f_ext = rng.normal(size=(n_fib, 3))
    ft = rng.normal(size=(2, 6))
    got = dict(fb=[], site=[], vg=[], fs=[], lp=[], E=[], mc=[], fext=[])
    for g in range(world):
        part = capi.partition_query(fiber_n, n_shell, sum(body_n), world, g)
        fl = RecordingFlow(fiber_n, n_shell, body_n, part)
        s = distributed.RankStepper(fl, None, params, 0.9, part, fiber_body=fiber_body, site_ref=site_ref,
                                    v_growth=v_growth, force_scale=force_scale, device="cpu")
        info = s.step(0.02, f_external=f_ext, body_forces_torques=ft)
        assert info["converged"] == 1 and len(fl.calls) == 1
        c = fl.calls[0]
        f0, f1 = part[:2]
        off = fl._fiber_off
        assert np.array_equal(c["fiber_body"], fiber_body[f0:f1])
        assert np.array_equal(c["site_ref"], site_ref[f0:f1])
        assert np.array_equal(c["v_growth"], v_growth[f0:f1]) and np.array_equal(c["force_scale"], force_scale[f0:f1])
        lp, E, r, pen, beta, mc, ph = c["params"][:7]
        assert np.array_equal(lp, lengths[f0:f1]) and np.array_equal(E, params[1][f0:f1]) and r == 0.0125
        assert np.array_equal(mc, params[5][f0:f1]) and ph == 0
        assert c["params"][7] == 0.02 and c["params"][8] == 0.9
        if off[f1] > off[f0]:
            assert np.array_equal(c["f_external"].reshape(-1, 3), f_ext[off[f0]:off[f1]])
        else:
            assert c["d_f_external"] == 0
        assert np.array_equal(c["forces"].reshape(-1, 3), ft[:, :3])
        assert np.array_equal(c["torques"].reshape(-1, 3), ft[:, 3:])
        assert c["dense_matvec"] is None and c["dense_minv"] is None
        assert s.x.shape[0] == distributed.system_rows(part, fiber_n, n_shell, body_n).size
        for key, v in (("fb", c["fiber_body"]), ("site", c["site_ref"]), ("vg", c["v_growth"]),
                       ("fs", c["force_scale"]), ("lp", lp), ("E", E), ("mc", mc)):
            got[key].append(v)
        got["fext"].append(np.zeros((0, 3)) if c["f_external"] is None else c["f_external"].reshape(-1, 3))
    # the members' slices, in rank order, are the complete arrays
    for key, full in (("fb", fiber_body), ("site", site_ref), ("vg", v_growth), ("fs", force_scale),
                      ("lp", lengths), ("E", params[1]), ("mc", params[5]), ("fext", f_ext)):
        assert np.array_equal(np.concatenate(got[key]), full), key


def test_rank_stepper_without_forces_passes_no_pointers():
    fiber_n, _ = fibers(1)
    part = capi.partition_query(fiber_n, 0, 0, 2, 1)
    fl = RecordingFlow(fiber_n, 0, [], part)
    s = distributed.RankStepper(fl, None, (np.ones(len(fiber_n)), 1e-3, 0.0125, 500.0, 1.0, 0, 0), 0.9, part,
                                device="cpu")
    s.step(0.01)
    c = fl.calls[0]
    assert c["d_f_external"] == 0 and c["d_body_forces"] == 0 and c["d_body_torques"] == 0
    assert c["fiber_body"] is None and c["site_ref"] is None

"""Host-side checks of the whole-system calls on systems with an empty block (tests/test_gpu_system_edges.py runs them on
the device): the row partition of the member shapes (capi.partition_query, distributed.system_rows,
capi.group_body_pieces) tiles the solution vector once and gives the empty members empty ranges; the CPU restatements
(tests/system_reference.py, tests/system_rhs_reference.py) accept every empty block and reduce on it to what the
remaining blocks give alone; the body block of one sphere obeys Stokes' law and the rotlet's closed form; and the Python
entry points take zero-length arrays.  No GPU needed."""
import numpy as np
import pytest

import oracle as orc
import system_reference as sr
import system_rhs_reference as rr
from skellysim_b200 import capi, distributed
from test_gpu_group_system import rhs_inputs
from test_gpu_system_edges import MEMBER_SEED, MEMBERS, SINGLE, host_body_solve
from test_gpu_system_matvec import make_case

ETA, DT = 0.9, 1e-3
EMPTY = dict(n_fibers=0, n_shell=0, n_body_nodes=0, n_bodies=0)


def _shape(kw, seed=MEMBER_SEED):
    fib, shell, bodies, ops, links, M, Minv, x = make_case(seed, **kw)
    return fib, dict(shell, M=M, Minv=Minv), bodies, ops, links, x


@pytest.mark.parametrize("name", list(MEMBERS))
def test_member_shapes_partition_as_intended_and_tile_once(name):
    kw, want = MEMBERS[name]["kw"], MEMBERS[name]["parts"]
    fib, shell, bodies, ops, links, x = _shape(kw)
    fn, ns, nb = list(fib["n_nodes"]), shell["pos"].shape[0], bodies["pos"].shape[0]
    base = 4 * fib["pos"].shape[0] + 3 * ns
    for n_members, parts in want.items():
        got = [capi.partition_query(fn, ns, nb, n_members, g) for g in range(n_members)]
        assert got == parts, (n_members, got)
        rows = [distributed.system_rows(p, fn, ns, bodies["n_nodes"]) for p in parts]
        assert np.array_equal(np.sort(np.concatenate(rows)), np.arange(x.size))
        seen = np.zeros(x.size - base, dtype=int)
        for p, r in zip(parts, rows):
            pcs = capi.group_body_pieces(bodies["n_nodes"], p[4], p[5])
            glob = np.concatenate([np.arange(q[2]) + q[1] for q in pcs]) if len(pcs) else np.zeros(0, dtype=int)
            assert np.array_equal(glob, r[r >= base] - base)
            seen[glob] += 1
            if p[0] == p[1]:  # no own fiber: no fiber row
                assert not np.any(r < 4 * fib["pos"].shape[0])
            if p[4] == p[5]:  # no own body node: no body row, no piece
                assert pcs.shape == (0, 3) and not np.any(r >= base)
            if p[0] == p[1] and p[2] == p[3] and p[4] == p[5]:
                assert r.size == 0
        assert (seen == 1).all()
    # what each shape is there for
    p3 = want[3]
    if name == "M1":
        assert sum(p[0] == p[1] for p in p3) == 1
    if name == "M2":
        assert p3[2][2] == p3[2][3] and all(p[0] < p[1] for p in p3)
    if name == "M5":
        assert p3[2] == (0, 0, 2, 2, 2, 2)
    if name == "M2s":
        assert p3[2][2] == p3[2][3] and all(p[0] < p[1] for p in p3)
    if name == "M6s":
        assert p3[0][0] == p3[0][1] and p3[0][2] < p3[0][3]
    # the symmetric plan of a member needs >= 2 x 1024 fiber nodes (2 x sym_block_nodes, skb_matvec.cu)
    assert MEMBERS[name]["sym"] == (fib["pos"].shape[0] >= 2048)


@pytest.mark.parametrize("name", list(SINGLE) + [k for k, v in MEMBERS.items() if v["rhs"]] + ["empty"])
def test_the_restatements_accept_every_empty_block(name):
    kw = EMPTY if name == "empty" else SINGLE[name] if name in SINGLE else MEMBERS[name]["kw"]
    fib, shell, bodies, ops, links, x = _shape(kw)
    params, fparams, src = rhs_inputs(fib, bodies, ops, 5)
    nf, ns, n_b = fib["pos"].shape[0], shell["pos"].shape[0], len(bodies["n_nodes"])
    n_sol = 4 * nf + 3 * ns + sum(3 * n + 6 for n in bodies["n_nodes"])
    assert x.size == n_sol
    res, vel, ft = sr.system_apply_matvec(fib, shell, bodies, ops, links, shell["M"], x, ETA)
    pc = sr.system_apply_preconditioner(ops["A"], ops["n_nodes"], shell["Minv"] if ns else None, bodies["A"],
                                        bodies["n_nodes"], x)
    rhs = rr.system_rhs(fib, shell, bodies, fparams, ETA, DT, f_ext=src["f_ext"], ft=src["ft"], points=src["points"],
                        background=src["background"], v_growth=src["v_growth"], force_scale=src["force_scale"])[0]
    for v in (res, pc, rhs):
        assert v.shape == (n_sol,) and np.isfinite(v).all()
    if n_b == 0:  # no body part; the rest is the fiber and periphery operator alone
        assert ft.shape == (0, 6)
        x_f, x_s, _ = sr.split(x, nf, ns)
        res_f, v_all = orc.apply_matvec_fibers(fib, dict(shell, density=x_s.reshape(ns, 3)),
                                               dict(pos=np.zeros((0, 3)), normals=np.zeros((0, 3)),
                                                    density=np.zeros((0, 3)), centers=np.zeros((0, 3)),
                                                    forces=np.zeros((0, 3)), torques=np.zeros((0, 3))),
                                               ops, x_f, ETA, vel if len(fib["n_nodes"]) else None)
        assert np.array_equal(res[:4 * nf], res_f)
    if nf == 0:  # no link rows: no link force on any body; the preconditioner is the periphery's and the bodies'
        assert vel.shape == (0, 7) and not ft.any()
        x_b = x[3 * ns:]
        if ns:
            assert np.array_equal(pc[:3 * ns], shell["Minv"] @ x[:3 * ns])
        if n_b:
            _, sol_off = sr._body_offsets(bodies["n_nodes"])
            for b, A in enumerate(bodies["A"]):
                sl = slice(int(sol_off[b]), int(sol_off[b + 1]))
                assert np.allclose(pc[3 * ns:][sl], np.linalg.solve(A, x_b[sl]), rtol=0, atol=1e-12)
    if n_sol == 0:
        assert res.size == pc.size == rhs.size == 0
    node = 4 * nf + 3 * ns
    for n in bodies["n_nodes"]:  # six RHS rows exactly zero
        assert np.array_equal(rhs[node + 3 * n:node + 3 * n + 6], np.zeros(6))
        node += 3 * n + 6


# discretisation error of the Stokes drag with the Fibonacci sphere of tests/test_gpu_system_edges.py (R = 1, eta = 1),
# the host's dense solve: measured 4.2e-4, 1.5e-4, 3.0e-5, 4.0e-6 at n = 100, 200, 400, 800
# (nodes at z = 1 - (2 i + 1) / n, the golden angle apart).  Neither lattice variant tried -- nodes at the poles,
# z = 1 - 2 i / (n - 1), or the golden angle at i + 1/2 -- nor the sign of the normals does better; smaller figures
# (1.6e-6 at n = 400) have been quoted for this set-up but do not reproduce with these operators and this RHS
STOKES_BOUND = {100: 5e-4, 200: 2e-4, 400: 4e-5, 800: 5e-6}


def test_a_sphere_moves_by_stokes_law_on_the_host():
    F = np.array([0.3, -0.7, 0.2])
    errs = []
    for n, bound in STOKES_BOUND.items():
        A, x = host_body_solve(n, 1.0, 1.0, F, np.zeros(3))
        U = F / (6 * np.pi)
        e = np.linalg.norm(x[3 * n:3 * n + 3] - U) / np.linalg.norm(U)
        assert e <= bound, (n, e)
        assert np.linalg.cond(A) < 7.0  # a well-conditioned second-kind system
        errs.append(e)
    assert all(b < a for a, b in zip(errs, errs[1:]))  # converges


def test_a_sphere_turns_by_its_rotlet_on_the_host():
    n, R, eta, L = 400, 0.5, 0.7, np.array([0.2, 0.5, -0.4])
    _, x = host_body_solve(n, R, eta, np.zeros(3), L)
    W = L / (8 * np.pi * eta * R ** 3)
    assert np.linalg.norm(x[3 * n + 3:] - W) / np.linalg.norm(W) <= 1e-13
    assert np.linalg.norm(x[3 * n:3 * n + 3]) <= 1e-13 * np.linalg.norm(W)


def test_python_entry_points_take_zero_length_arrays():
    assert capi.partition_query([], 0, 0, 3, 2) == (0, 0, 0, 0, 0, 0)
    assert capi.group_body_pieces([], 0, 0).shape == (0, 3)
    assert distributed.system_rows((0, 0, 0, 0, 0, 0), [], 0, []).size == 0
    assert distributed.system_rows((0, 0, 2, 2, 2, 2), [], 2, [2]).size == 0
    p = capi.fiber_params(0, np.zeros(0), 2.5e-3, 0.0125, 500.0, 1.0, 0, 0)
    assert p.size == 0 and capi._params_ptr(p) is None
    assert capi.Flow._colmajor_concat([]).size == 0
    if capi.device_count() == 0:  # without a device the calls stop at the device, not at the empty arrays
        for make in (lambda: capi.Flow(0), lambda: capi.MultiFlow([0, 0])):
            with pytest.raises(capi.SkbError, match="error 3:"):
                make()

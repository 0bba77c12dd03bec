"""CPU tests of the row ownership of the multi-device whole-vector operator (skb_mflow_apply_system_matvec /
_preconditioner, include/skelly_b200_flow.h) and of its exchange of the bodies' link forces: every member owns its
fibers' and periphery rows, the 3 rows of each body node in its body rows [b0, b1), and the six rows [U; w] of every body
whose first node it holds (skellysim_b200.distributed.system_rows); the members' per-body partial forces and torques are
added in rank order (group_ft_reduce_kernel)."""
import numpy as np
import pytest

from skellysim_b200 import capi
from skellysim_b200.distributed import system_rows


def _random_shape(rng):
    fib = rng.integers(2, 40, size=rng.integers(0, 30))
    bodies = rng.integers(1, 60, size=rng.integers(0, 6))
    return fib, int(rng.integers(0, 50)), bodies


@pytest.mark.parametrize("seed", range(40))
def test_system_rows_tile_the_solution_vector_once(seed):
    rng = np.random.default_rng(seed)
    fib, n_shell, bodies = _random_shape(rng)
    n_sol = 4 * int(fib.sum()) + 3 * n_shell + int(np.sum(3 * bodies + 6))
    for n_members in range(1, 9):
        parts = [capi.partition_query(fib, n_shell, int(bodies.sum()), n_members, g) for g in range(n_members)]
        rows = [system_rows(p, fib, n_shell, bodies) for p in parts]
        for r in rows:
            assert np.all(np.diff(r) > 0)
        every = np.concatenate(rows) if rows else np.zeros(0, dtype=np.int64)
        assert every.size == n_sol, (n_members, every.size, n_sol)
        assert np.array_equal(np.sort(every), np.arange(n_sol))


@pytest.mark.parametrize("seed", range(20))
def test_six_rows_go_to_the_owner_of_the_first_node(seed):
    rng = np.random.default_rng(100 + seed)
    fib, n_shell, bodies = _random_shape(rng)
    if bodies.size == 0:
        bodies = np.array([7, 3])
    n_body = int(bodies.sum())
    base = 4 * int(fib.sum()) + 3 * n_shell
    first = np.concatenate([[0], np.cumsum(bodies)[:-1]])
    sol = base + np.concatenate([[0], np.cumsum(3 * bodies + 6)[:-1]])
    for n_members in range(1, 9):
        parts = [capi.partition_query(fib, n_shell, n_body, n_members, g) for g in range(n_members)]
        owner = {int(i): g for g, p in enumerate(parts) for i in system_rows(p, fib, n_shell, bodies)}
        for b, n in enumerate(bodies):
            node_owner = next(g for g, p in enumerate(parts) if p[4] <= first[b] < p[5])
            for k in range(6):
                assert owner[int(sol[b] + 3 * n + k)] == node_owner
            for i in range(n):  # node rows: the owner of the node
                g = next(g for g, p in enumerate(parts) if p[4] <= first[b] + i < p[5])
                assert all(owner[int(sol[b] + 3 * i + k)] == g for k in range(3))


def _container_sum(contrib, body_of, n_b):
    """body_sum_kernel: per body its bound fibers' contributions in container order, from 0.0"""
    out = np.zeros((n_b, 6))
    for f, b in enumerate(body_of):
        if b >= 0:
            out[b] += contrib[f]
    return out


@pytest.mark.parametrize("n_members", [1, 2, 3, 5, 8])
def test_rank_order_sum_of_partials_equals_the_direct_sum(n_members):
    rng = np.random.default_rng(7 + n_members)
    n_fibers, n_b = 97, 4
    body_of = np.where(rng.random(n_fibers) < 0.6, rng.integers(0, n_b, n_fibers), -1)
    body_of[:n_b] = np.arange(n_b)
    contrib = rng.normal(size=(n_fibers, 6)) * 10.0 ** rng.uniform(-3, 3, size=(n_fibers, 1))
    n_nodes = rng.integers(8, 64, n_fibers)
    direct = _container_sum(contrib, body_of, n_b)
    total = np.zeros((n_b, 6))
    for g in range(n_members):  # member g: its own fibers' partial, added in rank order starting from 0.0
        f0, f1 = capi.partition_query(n_nodes, 0, 0, n_members, g)[:2]
        total = total + _container_sum(contrib[f0:f1], body_of[f0:f1], n_b)
    if n_members == 1:
        assert np.array_equal(total, direct)
    scale = np.zeros((n_b, 6))
    for f, b in enumerate(body_of):
        if b >= 0:
            scale[b] += np.abs(contrib[f])
    k = int(np.bincount(body_of[body_of >= 0]).max()) + n_members
    assert np.all(np.abs(total - direct) <= k * 2.0 ** -53 * scale)

"""Host-side checks of the rank-per-GPU whole-vector calls (include/skelly_b200_flow.h skb_flow_group_*): the local
vector's rows (distributed.system_rows) and the piece table a member lays its body rows out by (skb_group_body_pieces)
tile the body part of the solution vector exactly once, bodies cut between members and members without body rows
included; and the new entry points refuse NULL handles with an error code.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

from skellysim_b200 import capi
from skellysim_b200.distributed import system_rows

SHAPES = [([300, 300], 4), ([200, 200, 200], 2), ([200, 200, 200], 4), ([2, 2], 3), ([1, 2, 85, 255, 256, 257, 511], 5),
          ([7], 3), ([3, 5, 1, 9], 8)]


@pytest.mark.parametrize("body_n,members", SHAPES)
def test_pieces_tile_the_body_part_once(body_n, members):
    fib, n_shell = [8, 16, 24], 10
    n_body, sol = int(sum(body_n)), int(sum(3 * n + 6 for n in body_n))
    base = 4 * sum(fib) + 3 * n_shell
    seen = np.zeros(sol, dtype=int)
    for g in range(members):
        part = capi.partition_query(fib, n_shell, n_body, members, g)
        pieces = capi.group_body_pieces(body_n, part[4], part[5])
        assert pieces.shape[0] <= 3
        rows = system_rows(part, fib, n_shell, body_n)
        body_rows = rows[rows >= base] - base
        # the pieces are the member's body rows in ascending order, packed from local offset 0
        local = np.concatenate([np.arange(p[2]) + p[0] for p in pieces]) if len(pieces) else np.zeros(0, int)
        glob = np.concatenate([np.arange(p[2]) + p[1] for p in pieces]) if len(pieces) else np.zeros(0, int)
        assert np.array_equal(local, np.arange(body_rows.size))
        assert np.array_equal(glob, body_rows)
        seen[glob] += 1
    assert (seen == 1).all()


def test_bodies_cut_between_members_and_a_member_without_body_rows():
    # two bodies of 200 over two members: the cut is inside body 1; its six rows go with its first node
    p = capi.group_body_pieces([200, 200, 200], 0, 300)
    assert p.tolist() == [[0, 0, 606 + 300], [906, 1206, 6]]
    p = capi.group_body_pieces([200, 200, 200], 300, 600)
    assert p.tolist() == [[0, 906, 300], [300, 1212, 606]]
    # the tiny_bodies shape over three members: the last one owns no body rows
    parts = [capi.partition_query([8, 16] * 12, 300, 4, 3, g) for g in range(3)]
    assert parts[2][4] == parts[2][5]
    assert capi.group_body_pieces([2, 2], parts[2][4], parts[2][5]).shape == (0, 3)
    # a member inside one body: its node rows only, the six rows are the first node's owner's
    assert capi.group_body_pieces([10], 3, 6).tolist() == [[0, 9, 9]]
    # the three-piece case: tail of a cut body, the whole body and the head of the next, that body's six rows
    assert capi.group_body_pieces([4, 4, 4], 2, 10).tolist() == [[0, 6, 6], [6, 18, 24], [30, 48, 6]]


def test_body_pieces_refuse_bad_arguments():
    n = (C.c_int * 2)(2, 2)
    out = (C.c_int64 * 9)()
    k = C.c_int(0)
    L = capi.library()
    assert L.skb_group_body_pieces(n, 2, 3, 1, out, 3, C.byref(k)) != 0  # end < begin
    assert L.skb_group_body_pieces(None, 2, 0, 4, out, 3, C.byref(k)) != 0
    assert L.skb_group_body_pieces(n, 2, 0, 4, out, 0, C.byref(k)) != 0  # no room
    bad = (C.c_int * 2)(2, 0)
    assert L.skb_group_body_pieces(bad, 2, 0, 2, out, 3, C.byref(k)) != 0


def test_new_entry_points_refuse_null_handles():
    L = capi.library()
    n = (C.c_int * 1)(4)
    w = (C.c_double * 12)()
    assert L.skb_flow_group_set_body_operators(None, n, 1, w, w, w, w, None) != 0
    assert L.skb_flow_group_set_fiber_links(None, None, None, None) != 0
    assert L.skb_flow_group_apply_system_matvec_device(None, None, None, 1.0, None, None) != 0
    assert L.skb_flow_group_apply_system_preconditioner_device(None, None, None, None, None) != 0
    assert L.skb_flow_group_build_system_rhs_device(None, None, None, None, None, None, None, 1e-3, 1.0, None,
                                                    None) != 0

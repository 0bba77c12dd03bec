"""GPU tests of rigid bodies placed on the device (include/skelly_b200_flow.h skb_flow_set_body_frames / _place_bodies /
_get_body_operators and their skb_mflow_ / skb_flow_group_ twins; body_place_kernel): the placed inverse Q A_0^-1 Q^T
and E_i = R E_i,0 R^T held entry by entry to the extended-precision restatement tests/body_placement_reference.py
(|dev - ext| <= K_PLACE u S; tests/test_body_placement_cpu.py shows the criterion attainable and sharp), an identity
placement and a placement after 100 others bitwise the frames, a real body's placed operators against the host's
recomputation at the placement, skb_mflow and one rank per GPU bitwise the single device, and the refusals."""
import numpy as np
import pytest

import body_placement_reference as bp
import skellysim_b200 as skb
import system_reference as sr
from conftest import rel_max
from test_gpu_group_system import Members
from test_gpu_mflow_system import case, setup_mflow
from test_gpu_system_matvec import TOL, make_case, setup_flow

pytestmark = pytest.mark.gpu
ETA = 0.9
IDENTITY = np.array([1.0, 0.0, 0.0, 0.0])


def frames_of(bodies):
    """the body frames of a test case's bodies: nodes relative to their centre, the case's operators as the frame's"""
    off = np.concatenate([[0], np.cumsum(bodies["n_nodes"])]).astype(int)
    ref = np.concatenate([bodies["pos"][off[b]:off[b + 1]] - bodies["centers"][b]
                          for b in range(len(bodies["n_nodes"]))]) if len(off) > 1 else np.zeros((0, 3))
    inv = bodies.get("A_inv") or [np.linalg.inv(A) for A in bodies["A"]]
    return (bodies["n_nodes"], ref, bodies["normals"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"], inv)


def placed_geometry(frames, centers, qs):
    """the nodes and normals place_bodies forms on the host"""
    n_nodes, ref, nrm = frames[0], frames[1], frames[2]
    off = np.concatenate([[0], np.cumsum(n_nodes)]).astype(int)
    out = [bp.placed_geometry(ref[off[b]:off[b + 1]], nrm[off[b]:off[b + 1]], centers[b], qs[b])
           for b in range(len(n_nodes))]
    return np.concatenate([p for p, _ in out]), np.concatenate([n for _, n in out])


def _place(fl, centers, qs, links):
    fl.place_bodies(centers, qs)
    fl.set_fiber_links(links["body"], links["site"], links["rigidity"])


def _bodies_only(fl, pos, nrm, centers):
    fl.set_fibers(np.zeros((0, 3)), [], [])
    fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
    fl.set_bodies(pos, nrm, centers)
    fl.set_fiber_operators([], [], np.zeros((0, 3)), [], [])
    fl.set_fiber_preconditioner([])


def _random_frames(seed, sizes, scale_spread=3):
    rng = np.random.default_rng(seed)
    nb = int(sum(sizes))
    e = rng.normal(size=(nb, 3))
    e /= np.linalg.norm(e, axis=1)[:, None]
    E = [rng.normal(size=(nb, 3)) * 10.0 ** rng.uniform(-scale_spread, scale_spread, (nb, 1)) for _ in range(3)]
    inv = [rng.normal(size=(3 * n + 6,) * 2) * 10.0 ** rng.uniform(-scale_spread, scale_spread, 3 * n + 6)[None, :]
           for n in sizes]
    centers = 2.0 * np.arange(len(sizes))[:, None] * np.array([1.0, 0.3, -0.2])
    return (list(sizes), 0.4 * e, e, rng.uniform(0.5, 1.5, nb), *E, inv), centers, rng


def test_placed_operators_entry_by_entry():
    sizes = [1, 42, 400, 2000, 7, 13]
    frames, centers, rng = _random_frames(81, sizes)
    qs = bp.random_quaternions(rng, len(sizes))
    c1 = centers + rng.uniform(-1, 1, centers.shape)
    with skb.Flow(0) as fl:
        _bodies_only(fl, *placed_geometry(frames, centers, [IDENTITY] * len(sizes)), centers)
        fl.set_body_frames(*frames)
        fl.place_bodies(c1, qs)
        got = fl.get_body_operators()
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
    worst_inv = worst_e = 0.0
    for b, n in enumerate(sizes):
        r = bp.ratio(got["A_inv"][b], bp.place_inverse(frames[7][b], qs[b]),
                     bp.place_inverse(frames[7][b], qs[b], absolute=True))
        sl = slice(off[b], off[b + 1])
        E0 = [a[sl] for a in frames[4:7]]
        rE = max(bp.ratio(g[sl], e, s).max() for g, e, s in
                 zip((got["ex"], got["ey"], got["ez"]), bp.place_E(*E0, qs[b]), bp.place_E(*E0, qs[b], absolute=True)))
        assert r.max() <= bp.K_PLACE and rE <= bp.K_PLACE, (n, r.max(), rE)
        worst_inv, worst_e = max(worst_inv, r.max()), max(worst_e, rE)
    print(f"\nplaced operators: inverse {worst_inv:.2f}, E {worst_e:.2f} (K {bp.K_PLACE})")


def test_body_at_the_shared_memory_limit():
    """[8446, 2] nodes (m = 25 344: the largest body the preconditioner's GEMV admits): the placed inverse's columns,
    read through the preconditioner on unit vectors (a GEMV on e_j returns column j exactly), meet the bound on the
    first, a middle and the two [U; w] column tiles.  [8447, 1] is refused and leaves the placed operators."""
    import torch
    n_ok = [8446, 2]
    m0 = 3 * n_ok[0] + 6
    rng = np.random.default_rng(82)
    total = sum(n_ok)
    e = rng.normal(size=(total, 3))
    e /= np.linalg.norm(e, axis=1)[:, None]
    centers = np.array([[0.0, 0.0, 0.0], [3.0, 0.0, 0.0]])
    w, ex, ey, ez = rng.uniform(0.5, 1.5, total), *(rng.normal(size=(total, 3)) for _ in range(3))
    m1 = 3 * n_ok[1] + 6
    buf = np.empty(m0 * m0 + m1 * m1)
    rng.random(out=buf)
    buf -= 0.5
    A0 = buf[:m0 * m0].reshape((m0, m0), order="F")
    q = bp.random_quaternions(rng, 2)
    tiles = [0, 1, 4000, m0 // 3 - 2, m0 // 3 - 1]
    cols = np.concatenate([np.arange(3 * J, 3 * J + 3) for J in tiles])
    dev = torch.device("cuda", 0)
    from skellysim_b200 import capi
    import ctypes as C
    L = capi.library()

    def set_frames(n):
        ni = np.array(n, dtype=np.int32)
        capi._check(L.skb_flow_set_body_frames(fl._h, ni.ctypes.data_as(C.POINTER(C.c_int)), 2, capi._p(0.4 * e),
                                               capi._p(e), capi._p(w), capi._p(ex), capi._p(ey), capi._p(ez),
                                               capi._p(buf)))

    with skb.Flow(0) as fl:
        _bodies_only(fl, *placed_geometry((n_ok, 0.4 * e, e), centers, [IDENTITY] * 2), centers)
        set_frames(n_ok)
        fl.place_bodies(centers, q)
        fl.set_fiber_links(None)
        X = torch.zeros((len(cols), m0 + m1), dtype=torch.float64, device=dev)
        Y = torch.zeros_like(X)
        X[torch.arange(len(cols)), torch.from_numpy(cols)] = 1.0
        for k in range(len(cols)):
            fl.apply_system_preconditioner_device(None, X[k].data_ptr(), Y[k].data_ptr())
        with pytest.raises(skb.SkbError, match="error 1:.*shared memory"):
            set_frames([8447, 1])
        y2 = torch.zeros_like(Y[0])
        fl.apply_system_preconditioner_device(None, X[0].data_ptr(), y2.data_ptr())
        torch.cuda.synchronize()
        got, again = Y.cpu().numpy()[:, :m0].T, y2.cpu().numpy()
    assert np.array_equal(again, Y.cpu().numpy()[0])
    r = bp.ratio(got, bp.place_column_tiles(A0, q[0], tiles), bp.place_column_tiles(A0, q[0], tiles, absolute=True))
    del A0, buf
    assert r.max() <= bp.K_PLACE, r.max()
    print(f"\nlargest body: sampled columns {r.max():.2f} (K {bp.K_PLACE})")


@pytest.fixture(scope="module")
def system_case():
    fib, shell, bodies, ops, links, M, Minv, x = make_case(83, n_fibers=30, n_shell=200, n_body_nodes=600, n_bodies=3)
    return fib, dict(shell, M=M, Minv=Minv), bodies, ops, links, x


def test_identity_placement_is_the_frames_bitwise(system_case):
    fib, shell, bodies, ops, links, x = system_case
    frames = frames_of(bodies)
    c = bodies["centers"]
    ident = [IDENTITY] * len(c)
    pos, nrm = placed_geometry(frames, c, ident)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn, skb.Flow(0) as ref, skb.Dense(device_ids=[0]) as dr:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        fl.set_body_frames(*frames)
        _place(fl, c, ident, links)
        got = fl.get_body_operators()
        setup_flow(ref, dr, fib, shell, dict(bodies, pos=pos, normals=nrm), ops, links)
        r = (fl.apply_system_matvec(x, ETA, dense=dn), fl.apply_system_preconditioner(x, dense=dn))
        r_ref = (ref.apply_system_matvec(x, ETA, dense=dr), ref.apply_system_preconditioner(x, dense=dr))
    for k, a in enumerate(("ex", "ey", "ez")):
        assert np.array_equal(got[a], frames[4 + k])
    assert all(np.array_equal(g, f) for g, f in zip(got["A_inv"], frames[7]))
    assert np.array_equal(r[0], r_ref[0]) and np.array_equal(r[1], r_ref[1])


def test_no_drift_over_100_placements(system_case):
    fib, shell, bodies, ops, links, x = system_case
    frames = frames_of(bodies)
    c = bodies["centers"]
    rng = np.random.default_rng(84)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        fl.set_body_frames(*frames)
        _place(fl, c, [IDENTITY] * len(c), links)
        first = fl.apply_system_matvec(x, ETA, dense=dn)
        for _ in range(100):
            fl.place_bodies(c + rng.uniform(-0.5, 0.5, c.shape), bp.random_quaternions(rng, len(c)))
        _place(fl, c, [IDENTITY] * len(c), links)
        got = fl.get_body_operators()
        last = fl.apply_system_matvec(x, ETA, dense=dn)
    assert all(np.array_equal(got[a], frames[4 + k]) for k, a in enumerate(("ex", "ey", "ez")))
    assert all(np.array_equal(g, f) for g, f in zip(got["A_inv"], frames[7]))
    assert np.array_equal(first, last)


def test_real_body_against_host_recomputation():
    """sphere nodes with quadrature weights: the body placed on the device against the host's singularity_vectors,
    body_operator and inverse at the placement, uploaded through set_body_operators"""
    r0, n0, w = bp.sphere_body(400)
    E0 = sr.singularity_vectors(r0, n0, w)
    A0 = sr.body_operator(r0, n0, np.zeros(3), w, *E0)
    rng = np.random.default_rng(85)
    q, c = bp.random_quaternions(rng, 1), rng.uniform(-2, 2, (1, 3))
    pos, nrm = bp.placed_geometry(r0, n0, c[0], q[0])
    E1 = sr.singularity_vectors(pos, nrm, w)
    A1 = sr.body_operator(pos, nrm, c[0], w, *E1)
    x = rng.normal(size=A1.shape[0])
    with skb.Flow(0) as fl, skb.Flow(0) as host:
        _bodies_only(fl, r0, n0, np.zeros((1, 3)))
        fl.set_body_frames([400], r0, n0, w, *E0, [np.linalg.inv(A0)])
        fl.place_bodies(c, q)
        fl.set_fiber_links(None)
        _bodies_only(host, pos, nrm, c)
        host.set_body_operators([400], w, *E1, [np.linalg.inv(A1)])
        host.set_fiber_links(None)
        mv, mv_host = fl.apply_system_matvec(x, ETA), host.apply_system_matvec(x, ETA)
        y, y_host = fl.apply_system_preconditioner(x), host.apply_system_preconditioner(x)
    err = rel_max(mv, mv_host)
    res = np.linalg.norm(A1 @ y - x) / np.linalg.norm(x)
    res_host = np.linalg.norm(A1 @ y_host - x) / np.linalg.norm(x)
    print(f"\nreal body (400 nodes): matvec rows {err:.2e} relative to the host recomputation; preconditioner "
          f"residual {res:.2e} (host inverse {res_host:.2e})")
    assert err <= TOL, err
    assert res <= 10 * res_host, (res, res_host)


@pytest.mark.parametrize("devs", [[0], [0, 0]])
def test_mflow_places_bitwise_as_the_single_device(devs):
    """skb_mflow placing its bodies gives bitwise what it gives with the single device's placed operators uploaded
    (and, on one device, what the single flow gives)"""
    fib, shell, bodies, ops, links, M, Minv, x = case("40", 86)
    frames = frames_of(bodies)
    rng = np.random.default_rng(87)
    c1 = bodies["centers"] + rng.uniform(-0.2, 0.2, bodies["centers"].shape)
    qs = bp.random_quaternions(rng, len(c1))
    pos, nrm = placed_geometry(frames, c1, qs)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        fl.set_body_frames(*frames)
        _place(fl, c1, qs, links)
        single = (fl.apply_system_matvec(x, ETA, dense=dn), fl.apply_system_preconditioner(x, dense=dn))
        placed = fl.get_body_operators()
    with skb.MultiFlow(devs) as mf:
        setup_mflow(mf, fib, shell, bodies, ops, links)
        mf.set_body_frames(*frames)
        _place(mf, c1, qs, links)
        multi = (mf.apply_system_matvec(x, ETA), mf.apply_system_preconditioner(x))
    uploaded = dict(bodies, pos=pos, normals=nrm, centers=c1, ex=placed["ex"], ey=placed["ey"], ez=placed["ez"],
                    A_inv=placed["A_inv"])
    with skb.MultiFlow(devs) as mf:
        setup_mflow(mf, fib, shell, dict(uploaded, A=[np.linalg.inv(a) for a in placed["A_inv"]]), ops, links)
        mf.set_body_operators(bodies["n_nodes"], bodies["weights"], placed["ex"], placed["ey"], placed["ez"],
                              placed["A_inv"])
        mf.set_fiber_links(links["body"], links["site"], links["rigidity"])
        up = (mf.apply_system_matvec(x, ETA), mf.apply_system_preconditioner(x))
    assert np.array_equal(multi[0], up[0]) and np.array_equal(multi[1], up[1])
    if len(devs) == 1:
        assert np.array_equal(single[0], multi[0]) and np.array_equal(single[1], multi[1])


def test_group_members_place_bitwise_as_mflow():
    fib, shell, bodies, ops, links, M, Minv, x = case("40", 88)
    frames = frames_of(bodies)
    rng = np.random.default_rng(89)
    c1 = bodies["centers"] + rng.uniform(-0.2, 0.2, bodies["centers"].shape)
    qs = bp.random_quaternions(rng, len(c1))
    devs = [0, 0]
    with skb.MultiFlow(devs) as mf:
        setup_mflow(mf, fib, shell, bodies, ops, links)
        mf.set_body_frames(*frames)
        _place(mf, c1, qs, links)
        ref = (mf.apply_system_matvec(x, ETA), mf.apply_system_preconditioner(x))
    with skb.Flow(0) as fl:
        _bodies_only(fl, *placed_geometry(frames, bodies["centers"], [IDENTITY] * len(c1)), bodies["centers"])
        fl.set_body_frames(*frames)
        fl.place_bodies(c1, qs)
        single_ops = fl.get_body_operators()
    g = Members(devs, fib, shell, bodies, ops, links)
    try:
        for k, fl in enumerate(g.flows):
            f0, f1 = g.parts[k][:2]
            fl.group_set_body_frames(*frames)
            fl.group_place_bodies(c1, qs)
            fl.group_set_fiber_links(links["body"][f0:f1], links["site"][f0:f1], links["rigidity"][f0:f1])
        for fl in g.flows:
            got = fl.get_body_operators()
            assert all(np.array_equal(got[a], single_ops[a]) for a in ("ex", "ey", "ez"))
            assert any(a is not None for a in got["A_inv"])
            assert all(a is None or np.array_equal(a, s) for a, s in zip(got["A_inv"], single_ops["A_inv"]))
        res = (g.matvec(x), g.precondition(x))
        assert g.errors() == [-1] * len(devs)
    finally:
        g.close()
    assert np.array_equal(res[0], ref[0]) and np.array_equal(res[1], ref[1])


def _refused(call, match="error 1:"):
    with pytest.raises(skb.SkbError, match=match):
        call()


def test_refusals_and_edge_cases(system_case):
    fib, shell, bodies, ops, links, x = system_case
    frames = frames_of(bodies)
    c = bodies["centers"]
    rng = np.random.default_rng(90)
    qs = bp.random_quaternions(rng, len(c))
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        _refused(lambda: fl.place_bodies(c, qs), "set_body_frames first")
        fl.set_body_frames(*frames)
        _place(fl, c, qs, links)
        r0 = fl.apply_system_matvec(x, ETA, dense=dn)
        for bad in ([np.nan, 0, 0, 0], [np.inf, 0, 0, 0], [1.0 + 1e-11, 0, 0, 0], [0.5, 0.5, 0.5, 0.4]):
            q = qs.copy()
            q[1] = bad
            _refused(lambda: fl.place_bodies(c, q), "unit quaternion")
        assert np.array_equal(fl.apply_system_matvec(x, ETA, dense=dn), r0)  # refusals left the placement
        fl.place_bodies(c, qs * (1 + 4e-13))  # within the tolerance
        # skb_flow_set_bodies with other node counts: the frames no longer fit
        n = bodies["n_nodes"]
        fl.set_bodies(bodies["pos"][:-5], bodies["normals"][:-5], c)
        _refused(lambda: fl.place_bodies(c, qs), "frames")
        fl.set_bodies(bodies["pos"][:sum(n[:2])], bodies["normals"][:sum(n[:2])], c[:2])
        _refused(lambda: fl.place_bodies(c[:2], qs[:2]), "frames")
    with skb.Flow(0) as fl:  # no bodies: frames and placements of nothing
        _bodies_only(fl, np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_body_frames([], np.zeros((0, 3)), np.zeros((0, 3)), [], *(np.zeros((0, 3)),) * 3, [])
        fl.place_bodies(np.zeros((0, 3)), np.zeros((0, 4)))
        got = fl.get_body_operators()
        assert got["ex"].shape == (0, 3) and got["A_inv"] == []

"""GPU tests of the body block, the fiber-body links and the body preconditioner (body_ops.cuh, skb_body.cu) entry by
entry against the extended-precision restatement tests/body_block_reference.py: |dev - ext| <= K u S, K fixed in advance
(body_block_reference's docstring derives each; tests/test_body_block_ext_cpu.py shows the criterion attainable by a
float64 evaluation and failed by every planted defect).  Each kernel is isolated through the public API:

  * links: zero A_ and force_operator_, zero periphery and body densities.  Then the boundary rows 4n-14+t of res_fibers
    are the device's link[t] for t in {0, 1, 2, 4, 5, 6} (MODE 2 adds v_boundary to a zero sum), and row 3 is link[3] +
    v_0 . xs_0, v_0 the centre flow at the fiber's first node;
  * body forces and torques: the same, with U = omega = 0: the body node rows of res are then the flow v at the nodes,
    the centre Stokeslet of F and rotlet of L -- n_bodies sources per row -- held to ext F and L;
  * body_matvec_kernel: no links (F = L = 0); its rows are held to ext body_matvec on the device's own v_bodies;
  * the body preconditioner: every row to ext A_inv x, S = |A_inv| |x|, up to the largest body its GEMV admits.

Shapes: 40 bodies of 1, 2, 85, 255, 256, 257, 511, 513, 2000 and 3 .. 40 nodes, one with no fiber bound; fibers of
8, 31, 32, 33, 64, 96, 128 nodes, free ones first, 60 on one body; nucleation sites at |s| = 1e-6 .. 1e2; weights over
1e-3 .. 1e3.  The whole-vector operator is also held to tests/system_reference.py at the project's 1e-12 gate at the sizes
where the symmetric and cross kernels and the background dense streamer run, per body as well as per block.

Worst device ratio |dev - ext| / (u S) measured on an H100 80GB HBM3 (400 W power limit), against its K:
    link rows 0-2, 4-6: 2.33 (K 14)                  link row 3: 1.02, 0.006 of K
    body node rows (flow of F and L): 3.78, 0.025 of K (K 149)
    body_matvec node rows: 3.65 (K 14)               K^T lambda rows: 0.094 of K
    preconditioner rows: 0.17 of K                   largest body (m = 25 344, sampled rows): 0.46 (K 3179)
The largest-body test took 4.2 to 4.6 s there (about 5.1 GB of host and of device memory); the file, under 20 s.
"""
import ctypes as C

import numpy as np
import pytest

import body_block_reference as bb
import skellysim_b200 as skb
import system_reference as sr
from conftest import rel_max
from oracle.fiber_fd import compute_matrices
from skellysim_b200 import capi
from test_body_block_ext_cpu import BODY_NODES, FIBER_NODES, body_case, body_x, k_ft_per_body
from test_gpu_system_matvec import TOL, _check, blocks, make_case, setup_flow

pytestmark = pytest.mark.gpu
ETA = 0.9
N_SHELL = 64


def _ext_flow(r, bodies, fte, fts):
    c = bodies["centers"]
    return (bb.centre_flow(r, c, fte[:, :3], fte[:, 3:], ETA),
            bb.centre_flow(r, c, fts[:, :3], fts[:, 3:], ETA, absolute=True))


def _open(fl, dn, fib, ops, links, bodies, real, rng):
    """a flow whose fibers carry zero A_ and force_operator_ (uploaded; with real=True the tangents are the ones
    build_fiber_operators made from the positions), a periphery of N_SHELL nodes with a random dense operator, the
    bodies' operators without A_inv, and the links"""
    d = rng.normal(size=(N_SHELL, 3))
    d /= np.linalg.norm(d, axis=1)[:, None]
    fl.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
    fl.set_periphery(d * np.array([7.8, 4.16, 4.16]), -d)
    fl.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])
    for n in sorted(ops["D_2_0"]):
        if real:
            m = compute_matrices(n)
            D1, P, D4 = m["D_1_0"], m["P_downsample_bc"], m["D_4_0"]
        else:
            D1, P, D4 = rng.normal(size=(n, n)), rng.normal(size=(4 * n - 14, 4 * n)), rng.normal(size=(n, n))
        fl.set_fiber_class(n, D1, P)
        fl.set_fiber_class_derivatives(n, ops["D_2_0"][n], ops["D_3_0"][n], D4)
    nfib = len(fib["n_nodes"])
    if real:
        fl.build_fiber_operators(ops["length_prev"], 0.02, 0.0125, 500.0, 1.0, 0, 0, 1e-3, ETA)
        ops["xs"] = fl.get_fiber_operators(inverse=False)["xs"]
    fl.set_fiber_operators([np.zeros((4 * n, 4 * n)) for n in fib["n_nodes"]],
                           [np.zeros((3 * n, 4 * n)) for n in fib["n_nodes"]], ops["xs"], ops["length_prev"],
                           [0] * nfib)
    fl.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"])
    fl.set_fiber_links(links["body"], links["site"], links["rigidity"])
    dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, rng.normal(size=(3 * N_SHELL,) * 2))


@pytest.mark.parametrize("operators", ["uploaded", "built"])
def test_links_and_body_sums_entry_by_entry(operators):
    real = operators == "built"
    fnodes = tuple(n for n in FIBER_NODES if n % 8 == 0) if real else FIBER_NODES   # the build's node counts
    fib, ops, links, bodies = body_case(71, fiber_nodes=fnodes, real=real)
    rng = np.random.default_rng(72)
    nf, n_b = fib["pos"].shape[0], len(bodies["n_nodes"])
    x_f = rng.normal(size=4 * nf)
    x_moving = np.concatenate([x_f, np.zeros(3 * N_SHELL), body_x(rng, bodies, densities=False)])
    x_still = np.concatenate([x_f, np.zeros(3 * N_SHELL), body_x(rng, bodies, densities=False, motion=False)])
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        _open(fl, dn, fib, ops, links, bodies, real, rng)
        res_moving = fl.apply_system_matvec(x_moving, ETA, dense=dn)
        res_still = fl.apply_system_matvec(x_still, ETA, dense=dn)
    x_b = x_moving[4 * nf + 3 * N_SHELL:]
    le, _, fte = bb.link_terms(fib, ops, links, bodies, x_f, x_b)
    ls, _, fts = bb.link_terms(fib, ops, links, bodies, x_f, x_b, absolute=True)
    assert np.count_nonzero(fte[:-1].astype(np.float64)) == 6 * (n_b - 1) and not fte[-1].any()
    k_ft = k_ft_per_body(links, fib, n_b).max()
    k_v = bb.k_flow(n_b) + k_ft

    # the link rows of every fiber (free ones: exact zeros)
    first = np.concatenate([[0], np.cumsum(fib["n_nodes"])[:-1]]).astype(int)
    rows = np.array([4 * o + 4 * n - 14 for o, n in zip(first, fib["n_nodes"])])
    t = np.array([0, 1, 2, 4, 5, 6])
    r_link = bb.ratio(res_moving[rows[:, None] + t[None, :]], le[:, t], ls[:, t])
    assert r_link.max() <= bb.K_LINK_ROWS, (np.unravel_index(r_link.argmax(), r_link.shape), r_link.max())
    # row 3: link[3] + v_0 . xs_0
    v0e, v0s = _ext_flow(fib["pos"][first], bodies, fte, fts)
    xs0 = ops["xs"][first].astype(np.longdouble)
    e3 = le[:, 3] + np.sum(v0e * xs0, axis=1)
    s3 = ls[:, 3] + np.sum(v0s * np.abs(xs0), axis=1)
    k3 = bb.K_LINK_ROWS + k_v + 3
    r3 = bb.ratio(res_moving[rows + 3], e3, s3)
    assert r3.max() <= k3, (r3.argmax(), r3.max(), k3)

    # U = omega = 0, zero densities: the body node rows are the centre flow of F and L; the six rows are zero
    ve, vs = _ext_flow(bodies["pos"], bodies, fte, fts)
    g_b = blocks(res_still, fib, dict(pos=np.zeros((N_SHELL, 3))))[2]
    node_rows, six = [], []
    off = 0
    for n in bodies["n_nodes"]:
        node_rows.append(g_b[off:off + 3 * n])
        six.append(g_b[off + 3 * n:off + 3 * n + 6])
        off += 3 * n + 6
    r_v = bb.ratio(np.concatenate(node_rows), ve.reshape(-1), vs.reshape(-1))
    assert r_v.max() <= k_v, (r_v.argmax(), r_v.max(), k_v)
    assert not np.concatenate(six).any()
    print(f"\n{operators}: link rows {r_link.max():.2f} (K {bb.K_LINK_ROWS}), row 3 {r3.max() / k3:.3f} of K "
          f"({r3.max():.2f}), body node rows {r_v.max() / k_v:.3f} of K ({r_v.max():.2f}, K {k_v})")


def test_body_matvec_rows_entry_by_entry():
    import torch
    fib, ops, links, bodies = body_case(73)
    rng = np.random.default_rng(74)
    nf, nb, n_b = fib["pos"].shape[0], bodies["pos"].shape[0], len(bodies["n_nodes"])
    x_f, x_s, x_b = rng.normal(size=4 * nf), rng.normal(size=3 * N_SHELL), body_x(rng, bodies)
    x = np.concatenate([x_f, x_s, x_b])
    dens = np.concatenate([x_b[o:o + 3 * n] for o, n in
                           zip(np.concatenate([[0], np.cumsum(3 * np.array(bodies["n_nodes"]) + 6)[:-1]]),
                               bodies["n_nodes"])]).reshape(nb, 3)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        _open(fl, dn, fib, ops, links, bodies, False, rng)
        fl.set_fiber_links(None)
        d_x, d_res = t(x), torch.zeros(x.size, dtype=torch.float64, device=dev)
        fl.apply_system_matvec_device(dn, d_x.data_ptr(), ETA, d_res.data_ptr())
        zeros = t(np.zeros((n_b, 3)))
        r_f, r_s, v_b = (torch.zeros(k, dtype=torch.float64, device=dev) for k in (4 * nf, 3 * N_SHELL, 3 * nb))
        d_xf, d_xs, d_dens = t(x_f), t(x_s), t(dens)
        fl.apply_matvec_device(dn, d_xf.data_ptr(), d_xs.data_ptr(), d_dens.data_ptr(), zeros.data_ptr(),
                               zeros.data_ptr(), 0, ETA, r_f.data_ptr(), r_s.data_ptr(), v_b.data_ptr())
        torch.cuda.synchronize()
        res, r_f, r_s, v_b = (a.cpu().numpy() for a in (d_res, r_f, r_s, v_b))
    g_f, g_s, g_b = blocks(res, fib, dict(pos=np.zeros((N_SHELL, 3))))
    assert np.array_equal(g_f, r_f) and np.array_equal(g_s, r_s)
    v_b = v_b.reshape(nb, 3)
    r = bb.ratio(g_b, *bb.ext_and_scale(bb.body_rows, bodies, v_b, x_b))
    worst_node = worst_kt = 0.0
    off = 0
    for n in bodies["n_nodes"]:
        worst_node = max(worst_node, r[off:off + 3 * n].max())
        worst_kt = max(worst_kt, r[off + 3 * n:off + 3 * n + 6].max() / bb.k_kt(n))
        off += 3 * n + 6
    assert worst_node <= bb.K_NODE and worst_kt <= 1.0, (worst_node, worst_kt)
    print(f"\nbody_matvec: node rows {worst_node:.2f} (K {bb.K_NODE}), K^T lambda rows {worst_kt:.3f} of K")


def _bodies_only(fl, bodies):
    fl.set_fibers(np.zeros((0, 3)), [], [])
    fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
    fl.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])
    fl.set_fiber_operators([], [], np.zeros((0, 3)), [], [])
    fl.set_fiber_preconditioner([])


def test_body_preconditioner_entry_by_entry():
    fib, ops, links, bodies = body_case(75, n_bodies=len(BODY_NODES))
    rng = np.random.default_rng(76)
    A = [rng.normal(size=(3 * n + 6,) * 2) * 10.0 ** rng.uniform(-3, 3, 3 * n + 6)[None, :] for n in BODY_NODES]
    x = rng.normal(size=sum(a.shape[0] for a in A))
    with skb.Flow(0) as fl:
        _bodies_only(fl, bodies)
        fl.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"], A)
        fl.set_fiber_links(None)
        y = fl.apply_system_preconditioner(x)
    worst, off = 0.0, 0
    for a in A:
        m = a.shape[0]
        r = bb.ratio(y[off:off + m], *bb.ext_and_scale(bb.gemv_rows, a, x[off:off + m]))
        worst = max(worst, r.max() / bb.k_gemv(m))
        assert r.max() <= bb.k_gemv(m), (m, r.argmax(), r.max(), bb.k_gemv(m))
        off += m
    print(f"\nbody preconditioner: {worst:.3f} of K")


def test_body_preconditioner_at_its_shared_memory_limit():
    """The GEMV keeps a body's x (its 3n + 6 unknowns, rounded up to even) and 256 slice partials in shared memory, at
    most 200 KB: the largest body it admits has n = 8446 nodes (m = 25 344).  Two bodies, [8446, 2] nodes: accepted,
    64 sampled rows of the big body and every row of the small one meet the entry-wise bound.  Then the same flow split
    as [8447, 1] is refused, and the operators set before still give bitwise the same result.  The inverses live in one
    column-major host buffer passed through the C ABI (about 5.1 GB on the host and on the device)."""
    import torch
    n_ok, n_bad = [8446, 2], [8447, 1]
    m0, m1 = 3 * n_ok[0] + 6, 3 * n_ok[1] + 6
    rng = np.random.default_rng(77)
    total = sum(n_ok)
    e = rng.normal(size=(total, 3))
    e /= np.linalg.norm(e, axis=1)[:, None]
    centers = np.array([[0.0, 0.0, 0.0], [3.0, 0.0, 0.0]])
    pos = np.concatenate([centers[0] + 0.4 * e[:n_ok[0]], centers[1] + 0.4 * e[n_ok[0]:]])
    w, ex, ey, ez = rng.uniform(0.5, 1.5, total), *(rng.normal(size=(total, 3)) for _ in range(3))
    buf = np.empty((3 * n_bad[0] + 6) ** 2 + (3 * n_bad[1] + 6) ** 2)
    rng.random(out=buf)
    buf -= 0.5
    A0 = buf[:m0 * m0].reshape((m0, m0), order="F")
    A1 = buf[m0 * m0:m0 * m0 + m1 * m1].reshape((m1, m1), order="F")
    x = rng.normal(size=m0 + m1)
    L = capi.library()

    def set_ops(n):
        ni = np.array(n, dtype=np.int32)
        capi._check(L.skb_flow_set_body_operators(fl._h, ni.ctypes.data_as(C.POINTER(C.c_int)), 2, capi._p(w),
                                                  capi._p(ex), capi._p(ey), capi._p(ez), capi._p(buf)))

    dev = torch.device("cuda", 0)
    with skb.Flow(0) as fl:
        _bodies_only(fl, dict(pos=pos, normals=e, centers=centers))
        set_ops(n_ok)
        d_x = torch.from_numpy(x).to(dev)
        d_y1, d_y2 = torch.zeros_like(d_x), torch.zeros_like(d_x)
        fl.apply_system_preconditioner_device(None, d_x.data_ptr(), d_y1.data_ptr())
        with pytest.raises(skb.SkbError, match="error 1:.*shared memory"):
            set_ops(n_bad)
        fl.apply_system_preconditioner_device(None, d_x.data_ptr(), d_y2.data_ptr())
        torch.cuda.synchronize()
        y1, y2 = d_y1.cpu().numpy(), d_y2.cpu().numpy()
    assert np.array_equal(y1, y2)
    rows = np.unique(np.concatenate([[0, 31, 32, 255, 256, m0 - 33, m0 - 32, m0 - 1],
                                     rng.choice(m0, 56, replace=False)]))[:64]
    r0 = bb.ratio(y1[rows], *bb.ext_and_scale(bb.gemv_rows, A0, x[:m0], rows))
    r1 = bb.ratio(y1[m0:], *bb.ext_and_scale(bb.gemv_rows, A1, x[m0:]))
    del A0, A1, buf
    assert r0.max() <= bb.k_gemv(m0) and r1.max() <= bb.k_gemv(m1), (r0.max(), r1.max())
    print(f"\nlargest body: {r0.max() / bb.k_gemv(m0):.3f} of K ({r0.max():.2f}, K {bb.k_gemv(m0)}); "
          f"small body {r1.max():.2f}")


@pytest.fixture(scope="module")
def fast_case():
    """150 fibers of 32 nodes (4800 fiber nodes: the symmetric kernel), 500 periphery nodes (the cross kernel and the
    background dense streamer), 2 bodies of 300 nodes, every other fiber bound"""
    fib, shell, bodies, ops, links, M, Minv, x = make_case(41, n_fibers=150, n_shell=500, n_body_nodes=600,
                                                           nodes=(32,))
    return fib, dict(shell, M=M, Minv=Minv), bodies, ops, links, M, x


def test_whole_vector_at_the_fast_path_sizes(fast_case):
    fib, shell, bodies, ops, links, M, x = fast_case
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        res = fl.apply_system_matvec(x, ETA, dense=dn)
        launches = fl.stats()["launches"]
        _, sym_pairs = fl.last_sym_kernel()
        again = fl.apply_system_matvec(x, ETA, dense=dn)
        fl.set_cross(0)
        no_cross = fl.apply_system_matvec(x, ETA, dense=dn)
        launches_no_cross = fl.stats()["launches"]
        fl.set_cross(-1)
        fl.set_overlap(False)
        no_overlap = fl.apply_system_matvec(x, ETA, dense=dn)
    assert sym_pairs > 0, "the symmetric kernel did not run"
    assert launches != launches_no_cross, "the cross kernel did not run"
    assert np.array_equal(res, again)
    ref, vel, ft = sr.system_apply_matvec(fib, shell, bodies, ops, links, M, x, ETA)
    assert np.count_nonzero(ft) > 0 and np.count_nonzero(vel) > 0
    for got in (res, no_cross, no_overlap):
        for got_b, ref_b in zip(blocks(got, fib, shell), blocks(ref, fib, shell)):
            _check(got_b, ref_b)
        g_b, r_b = blocks(got, fib, shell)[2], blocks(ref, fib, shell)[2]
        off = 0
        for n in bodies["n_nodes"]:  # each body's node rows and its six rows on their own
            for sl in (slice(off, off + 3 * n), slice(off + 3 * n, off + 3 * n + 6)):
                assert rel_max(g_b[sl], r_b[sl]) <= TOL, (n, sl, rel_max(g_b[sl], r_b[sl]))
            off += 3 * n + 6
    for other in (no_cross, no_overlap):
        for got_b, ref_b in zip(blocks(other, fib, shell), blocks(res, fib, shell)):
            assert rel_max(got_b, ref_b) <= TOL


def test_device_forms_on_a_side_stream_beside_a_busy_one(fast_case):
    import torch
    fib, shell, bodies, ops, links, M, x = fast_case
    dev = torch.device("cuda", 0)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        r_host = fl.apply_system_matvec(x, ETA, dense=dn)
        p_host = fl.apply_system_preconditioner(x, dense=dn)
        d_x = torch.from_numpy(x).to(dev)
        d_r, d_p = torch.zeros_like(d_x), torch.zeros_like(d_x)
        a = torch.randn(2048, 2048, dtype=torch.float64, device=dev)
        torch.cuda.synchronize()
        busy, side = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
        with torch.cuda.stream(busy):
            b = a
            for _ in range(16):
                b = (b @ a) / 64.0
        fl.apply_system_matvec_device(dn, d_x.data_ptr(), ETA, d_r.data_ptr(), stream=side.cuda_stream)
        fl.apply_system_preconditioner_device(dn, d_x.data_ptr(), d_p.data_ptr(), stream=side.cuda_stream)
        side.synchronize()
        r_dev, p_dev = d_r.cpu().numpy(), d_p.cpu().numpy()
        torch.cuda.synchronize()
        assert torch.isfinite(b).all()
    assert np.array_equal(r_dev, r_host) and np.array_equal(p_dev, p_host)

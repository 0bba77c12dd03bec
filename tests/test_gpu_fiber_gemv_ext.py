"""GPU tests of fiber_gemv_kernel<MODE> (fiber_ops.cuh; FiberOps::force / matvec / precondition in skb_fiber.cu) entry by
entry against the extended-precision restatement tests/fiber_gemv_reference.py: every device entry of every mode meets
|dev - ext| <= K u S, K fixed in advance (the reference's docstring derives each; tests/test_fiber_gemv_ext_cpu.py
shows the criterion attainable by a float64 evaluation and failed by every planted defect).  An entry with S = 0 must be
exact.

    MODE 1  skb_flow_apply_fiber_force          force_operator_ x, scattered into the Stokeslet strengths
    MODE 2  skb_flow_fiber_matvec               A_ x - P_downsample_bc vT(v) + xs_vT + y_BC
    MODE 0  skb_flow_apply_fiber_preconditioner A_^-1 x

Shapes: fibers of 4, 5, 7, 8, 14, 15, 16, 17, 31, 32, 33, 48, 64, 96 and 128 nodes, small and large alternating, with
x and v scaled per fiber over 1e-3 .. 1e3, length_prev over 1e-2 .. 1e2, plus_velocity mixed, v_boundary absent and
present; the flow's own fibers start mid-list (skb_flow_set_target_ranges with f0 > 0).  Operators: (a) dense random
stand-ins with an all-zero P row, a P row with zeros inside its range and an all-zero D_1_0 column; (b) the reference's
operators (P block diagonal, D_1_0 banded), clamp and pin fractions 0 and 0.5; (c) the device build on curved fibers of
8 .. 128 nodes, held to its own downloaded A_, force_operator_, xs_ and A_^-1.  Then the device-pointer forms on a side
stream, the fiber rows of skb_mflow_apply_system_preconditioner on two members, and one fiber of 2816 nodes, where the
kernel's dynamic shared memory, (9n + 256) x 8 bytes, is exactly the 200 KB the kernels allow; 2817 nodes are refused.

Worst device ratio |dev - ext| / (u S) as a fraction of its K, measured on an H100 80GB HBM3 (700 W power limit):
                          MODE 0   MODE 1   MODE 2
    (a) dense              0.105    0.077    0.033
    (b) clamp / pin 0      0.143    0.139    0.067
    (b) clamp / pin 0.5    0.118    0.123    0.066
    (c) device-built       0.098    0.139    0.084
    device forms           0.066    0.058    0.036
    mflow, members [0, 0]  0.071
At n = 2816, on the sampled rows, the ratios themselves are 0.74 in MODE 0 and 0.64 in MODE 1 (K 1419), 0.52 in MODE 2
(K 1789).  The n = 2816 test took 17.8 s there, with A_, force_operator_ and P (2.8 GB) on the host; the file, 26 s.
A P walk cut short by one column (the p_range_short defect edited into fiber_ops.cuh) fails
test_every_row_of_every_mode on its first family.
"""
import numpy as np
import pytest

import fiber_gemv_reference as fg
import skellysim_b200 as skb
from oracle import fiber_fd
from skellysim_b200 import capi
from test_fiber_gemv_ext_cpu import alternating, dense_case, inputs, reference_case
from test_gpu_fiber_build import curved_fibers

pytestmark = pytest.mark.gpu
ETA = 0.9
BUILD_NODES = (8, 16, 24, 32, 48, 64, 96, 128)   # the node counts the device build's own tests cover (8 <= n <= 128)
LIMIT_N = 2816                                   # (9 n + 256) x 8 B = 200 KB


def _own(ops, A_inv, x, v, vb, f0, f1):
    off = np.concatenate([[0], np.cumsum(ops["n_nodes"])]).astype(int)
    a, b = off[f0], off[f1]
    own = dict(ops, n_nodes=ops["n_nodes"][f0:f1], A=ops["A"][f0:f1], force=ops["force"][f0:f1], xs=ops["xs"][a:b],
               length_prev=ops["length_prev"][f0:f1], plus=ops["plus"][f0:f1])
    return own, A_inv[f0:f1], x[4 * a:4 * b], v[a:b], vb[f0:f1]


def _open(fl, fib, ops):
    fl.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
    fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
    fl.set_bodies(np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
    for n in sorted(ops["D_1_0"]):
        fl.set_fiber_class(n, ops["D_1_0"][n], ops["P"][n])


def _hold(worst, key, got, fn, args, K):
    r = fg.ratio(got, *fg.ext_and_scale(fn, *args))
    w = float(np.max(r / K))
    assert np.isfinite(r).all() and w <= 1.0, (key, np.unravel_index(np.argmax(r / K), r.shape), r.max())
    worst[key] = max(worst.get(key, 0.0), w)


def _hold_all(worst, family, own, Ai, x, v, vb, fw, res, res_vb, y):
    _hold(worst, (family, 1), fw, fg.fiber_force, (own["force"], x, own["n_nodes"]), fg.k_rows(own, 1))
    _hold(worst, (family, 2), res, fg.fiber_matvec, (own, x, v, None), fg.k_rows(own, 2))
    _hold(worst, (family, 2), res_vb, fg.fiber_matvec, (own, x, v, vb), fg.k_rows(own, 2))
    _hold(worst, (family, 0), y, fg.fiber_precondition, (Ai, x, own["n_nodes"]), fg.k_rows(own, 0))


def _report(worst):
    print("\n" + "; ".join(f"{fam} MODE {m}: {w:.3f} of K" for (fam, m), w in sorted(worst.items())))


FAMILIES = {"dense": lambda: dense_case(11, reps=3), "reference_0": lambda: reference_case(12, 0.0, 0.0, reps=3),
            "reference_half": lambda: reference_case(13, 0.5, 0.5, reps=3)}


@pytest.mark.parametrize("family", sorted(FAMILIES))
def test_every_row_of_every_mode(family):
    fib, ops, A_inv, x, v, vb = FAMILIES[family]()
    nfib = len(ops["n_nodes"])
    f0, f1 = 3, nfib - 2                                # own fibers start and end mid-list
    own, Ai, xo, vo, vbo = _own(ops, A_inv, x, v, vb, f0, f1)
    with skb.Flow(0) as fl:
        _open(fl, fib, ops)
        fl.set_target_ranges(f0, f1, 0, 0, 0, 0)
        fl.set_fiber_operators(own["A"], own["force"], own["xs"], own["length_prev"], own["plus"])
        fl.set_fiber_preconditioner(Ai)
        fw = fl.apply_fiber_force(xo)
        res, res_vb = fl.fiber_matvec(xo, vo), fl.fiber_matvec(xo, vo, vbo)
        y = fl.apply_fiber_preconditioner(xo)
    worst = {}
    _hold_all(worst, family, own, Ai, xo, vo, vbo, fw, res, res_vb, y)
    _report(worst)


def test_device_built_operators():
    """(c): A_, force_operator_, xs_ and A_^-1 from skb_flow_build_fiber_operators on curved fibers (own fibers from the
    second on), each mode held to the downloaded operators: the componentwise S makes the check independent of A_'s
    conditioning, so this is the entry-wise test of the applied preconditioner."""
    n_nodes = alternating(BUILD_NODES, 2)
    fib, prm = curved_fibers(21, n_nodes)
    rng = np.random.default_rng(22)
    x, v, vb = inputs(rng, n_nodes)
    f0, f1 = 1, len(n_nodes)
    with skb.Flow(0) as fl:
        fl.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
        fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_bodies(np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
        classes = {}
        for n in sorted(set(n_nodes)):
            m = fiber_fd.compute_matrices(n)
            classes[n] = m
            fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
            fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
        fl.set_target_ranges(f0, f1, 0, 0, 0, 0)
        fl.build_fiber_operators(*(prm[k][f0:f1] for k in ("length_prev", "bending_rigidity", "radius",
                                                           "penalty_param", "beta_tstep", "minus_clamped",
                                                           "plus_hinged")), 5e-3, ETA)
        got = fl.get_fiber_operators(inverse=True)
        off = np.concatenate([[0], np.cumsum(n_nodes)]).astype(int)
        a, b = off[f0], off[f1]
        xo, vo, vbo = x[4 * a:4 * b], v[a:b], vb[f0:f1]
        fw = fl.apply_fiber_force(xo)
        res, res_vb = fl.fiber_matvec(xo, vo), fl.fiber_matvec(xo, vo, vbo)
        y = fl.apply_fiber_preconditioner(xo)
    own = dict(n_nodes=n_nodes[f0:f1], A=got["A"], force=got["force"], xs=got["xs"],
               length_prev=list(prm["length_prev"][f0:f1]), plus=[int(p) for p in prm["plus_hinged"][f0:f1]],
               D_1_0={n: classes[n]["D_1_0"] for n in classes}, P={n: classes[n]["P_downsample_bc"] for n in classes})
    assert any(own["plus"]) and not all(own["plus"])
    worst = {}
    _hold_all(worst, "built", own, got["A_inv"], xo, vo, vbo, fw, res, res_vb, y)
    _report(worst)


def test_device_pointer_forms_on_a_side_stream_are_bitwise_the_host_forms():
    import torch
    fib, ops, A_inv, x, v, vb = dense_case(31, reps=1)
    f0, f1 = 2, len(ops["n_nodes"]) - 1
    own, Ai, xo, vo, vbo = _own(ops, A_inv, x, v, vb, f0, f1)
    n_own = vo.shape[0]
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    with skb.Flow(0) as fl:
        _open(fl, fib, ops)
        fl.set_target_ranges(f0, f1, 0, 0, 0, 0)
        fl.set_fiber_operators(own["A"], own["force"], own["xs"], own["length_prev"], own["plus"])
        fl.set_fiber_preconditioner(Ai)
        h = (fl.apply_fiber_force(xo), fl.fiber_matvec(xo, vo), fl.fiber_matvec(xo, vo, vbo),
             fl.apply_fiber_preconditioner(xo))
        d_x, d_v, d_vb = t(xo), t(vo), t(vbo)
        nan = lambda *s: torch.full(s, float("nan"), dtype=torch.float64, device=dev)
        d_fw, d_r, d_rvb, d_y = nan(n_own, 3), nan(4 * n_own), nan(4 * n_own), nan(4 * n_own)
        torch.cuda.synchronize()
        side = torch.cuda.Stream(dev)
        s = side.cuda_stream
        fl.apply_fiber_force_device(d_x.data_ptr(), d_fw.data_ptr(), s)
        fl.fiber_matvec_device(d_x.data_ptr(), d_v.data_ptr(), 0, d_r.data_ptr(), s)
        fl.fiber_matvec_device(d_x.data_ptr(), d_v.data_ptr(), d_vb.data_ptr(), d_rvb.data_ptr(), s)
        fl.apply_fiber_preconditioner_device(d_x.data_ptr(), d_y.data_ptr(), s)
        side.synchronize()
        d = tuple(a.cpu().numpy() for a in (d_fw, d_r, d_rvb, d_y))
    for got, want in zip(d, h):
        assert np.array_equal(got, want)
    worst = {}
    _hold_all(worst, "device forms", own, Ai, xo, vo, vbo, *d)
    _report(worst)


def test_fiber_rows_of_the_mflow_preconditioner():
    """the fiber rows of skb_mflow_apply_system_preconditioner (MODE 0 on every member, on the member's own fibers)
    for two members on one device, and on two devices when there are two"""
    fib, ops, A_inv, x, v, vb = dense_case(41, reps=2)
    lists = [[0, 0]] + ([[0, 1]] if capi.device_count() >= 2 else [])
    for devs in lists:
        with skb.MultiFlow(devs) as mf:
            mf.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
            mf.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
            mf.set_bodies(np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
            for n in sorted(ops["D_1_0"]):
                mf.set_fiber_class(n, ops["D_1_0"][n], ops["P"][n])
            mf.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
            mf.set_fiber_preconditioner(A_inv)
            mf.set_body_operators([], np.zeros(0), np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)), [])
            mf.set_fiber_links(None)
            parts = [mf.partition(g)[:2] for g in range(len(devs))]
            y = mf.apply_system_preconditioner(x)
        assert parts[0][0] == 0 and parts[0][1] == parts[1][0] > 0, parts     # the second member starts mid-list
        worst = {}
        _hold(worst, ("mflow", 0), y, fg.fiber_precondition, (A_inv, x, ops["n_nodes"]), fg.k_rows(ops, 0))
        print(f"\nmflow {devs}: MODE 0 {worst['mflow', 0]:.3f} of K")


# ---- the shared-memory limit ----

def _limit_case(rng):
    """one fiber of LIMIT_N nodes: D_1_0 banded (9 rows per column), P block diagonal with dense blocks as the
    reference's (three (n-4) x n, one (n-2) x n), all column-major"""
    n = LIMIT_N
    D = np.zeros((n, n), order="F")
    for k in range(-4, 5):
        i = np.arange(max(0, -k), min(n, n - k))
        D[i, i + k] = rng.normal(size=i.size)
    P = np.zeros((4 * n - 14, 4 * n), order="F")
    for s, h in enumerate((n - 4, n - 4, n - 4, n - 2)):
        r0 = s * (n - 4)
        P[r0:r0 + h, s * n:(s + 1) * n] = rng.normal(size=(h, n))
    return D, P


def _limit_rows(m, n):
    """the first and last row of every 32-row block (segments of n rows are whole blocks at n = 2816), and MODE 2's
    14 boundary rows"""
    r = np.arange(0, m, fg.ROWS)
    rows = np.concatenate([r, r + fg.ROWS - 1])
    if m == 4 * n:
        rows = np.concatenate([rows, np.arange(4 * n - 14, 4 * n)])
    return np.unique(rows)


def test_largest_fiber_and_the_refusal_past_it():
    """n = 2816: the kernels' dynamic shared memory is exactly 200 KB.  A_ (about 1 GB, also passed as the
    preconditioner's A_^-1: the GEMV is plain linear algebra), force_operator_ (0.76 GB) and P (1 GB) are dense random;
    sampled rows of every mode meet the bound.  Then n = 2817 is refused with SKB_ERR_INVALID before any launch, and
    setting the 2816-node operators again gives bitwise the same results.  (set_target_ranges drops the resident
    operators, as a refused set_fiber_operators does: the refusal leaves none behind, and the class table and the
    flow stay usable.)"""
    n = LIMIT_N
    rng = np.random.default_rng(51)
    pos = np.concatenate([np.linspace(0, 1, n)[:, None] * [0.0, 0.0, 1.0],
                          [2.0, 0.0, 0.0] + np.linspace(0, 1, n + 1)[:, None] * [0.0, 0.0, 1.0]])
    D, P = _limit_case(rng)
    xs = np.tile([0.0, 0.0, 1.0], (n, 1)) + 0.1 * rng.normal(size=(n, 3))
    xs /= np.linalg.norm(xs, axis=1)[:, None]
    lp, plus = 0.37, 1
    x = rng.normal(size=4 * n)
    v = rng.normal(size=(n, 3))
    vb = rng.normal(size=(1, 7))
    L = capi.library()

    def operators(seed):
        g = np.random.default_rng(seed)
        A, F = np.empty(16 * n * n), np.empty(12 * n * n)
        g.random(out=A)
        g.random(out=F)
        A -= 0.5
        F -= 0.5
        return A, F

    def set_ops(fl, A, F):
        fl.set_target_ranges(0, 1, 0, 0, 0, 0)
        fl.set_fiber_operators(A, F, xs, [lp], [plus], colmajor=True)
        capi._check(L.skb_flow_set_fiber_preconditioner(fl._h, capi._p(A)))

    def run(fl):
        return fl.apply_fiber_force(x), fl.fiber_matvec(x, v, vb), fl.apply_fiber_preconditioner(x)

    with skb.Flow(0) as fl:
        fl.set_fibers(pos, [n, n + 1], [1.0, 1.0])
        fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_bodies(np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_fiber_class(n, D, P)
        A, F = operators(52)
        set_ops(fl, A, F)
        fw, res, y = run(fl)
        Am = A.reshape((4 * n, 4 * n), order="F")
        Fm = F.reshape((3 * n, 4 * n), order="F")
        ra, rf = _limit_rows(4 * n, n), _limit_rows(3 * n, n)
        K0, K2 = fg.k_gemv(4 * n), fg.k_matvec_of(D, P)
        r1 = fg.ratio(fw.reshape(-1)[3 * (rf % n) + rf // n], *fg.ext_and_scale(fg.gemv, Fm, x, rf)) / K0
        r0 = fg.ratio(y[ra], *fg.ext_and_scale(fg.gemv, Am, x, ra)) / K0
        r2 = fg.ratio(res[ra], *fg.ext_and_scale(fg.matvec_rows, Am, D, P, xs, lp, plus, x, v, vb[0], ra)) / K2
        del A, F, Am, Fm, P
        assert max(r0.max(), r1.max(), r2.max()) <= 1.0, (r0.max(), r1.max(), r2.max())
        # one node more: refused before anything runs
        fl.set_fiber_class(n + 1, np.zeros((n + 1, n + 1)), np.zeros((4 * n - 10, 4 * n + 4), order="F"))
        fl.set_target_ranges(0, 2, 0, 0, 0, 0)
        before = capi.launch_count()
        with pytest.raises(skb.SkbError, match="error 1:.*2817 nodes exceeds the shared-memory"):
            fl.set_fiber_operators(np.zeros(1), np.zeros(1), np.zeros((2 * n + 1, 3)), [lp, lp], [plus, plus],
                                   colmajor=True)
        with pytest.raises(skb.SkbError, match="set_fiber_operators"):
            fl.apply_fiber_force(np.zeros(4 * (2 * n + 1)))
        assert capi.launch_count() == before
        A, F = operators(52)
        set_ops(fl, A, F)
        again = run(fl)
    for a, b in zip(again, (fw, res, y)):
        assert np.array_equal(a, b)
    print(f"\nn = {n}: MODE 0 {r0.max() * K0:.2f}, MODE 1 {r1.max() * K0:.2f} (K {K0}); MODE 2 {r2.max() * K2:.2f} "
          f"(K {K2})")

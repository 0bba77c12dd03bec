"""GPU tests of the whole-system calls (include/skelly_b200_flow.h skb_flow_apply_system_matvec / _preconditioner /
build_system_rhs, their _device forms, skb_mflow_* and skb_flow_group_*) on systems with an empty block: no fibers, no
periphery, no bodies, or nothing at all, on one device, and members of a group that own none of some block or nothing.
These are the shapes SkellySim is run in (a body alone, a body in a periphery, one clamped fiber, a periphery with point
sources, a nucleation start of bodies without fibers) and the shapes the row partition hands a member when a block is
smaller than the group.

Every result is held at the project's gate (1e-12 relative, max-norm and l2) per block and per body, for its node rows
and its six rows, to tests/system_reference.py and tests/system_rhs_reference.py; the six RHS rows of every body are
exactly +0.0.  Device outputs are filled with NaN first, so a row no launch writes fails.  Results are bitwise
reproducible and leave x untouched; the members' rows are bitwise those of one device.

The member shapes M1-M5 are small: every member takes the plain kernel for its own rows.  M2s, M3s and M6s have
>= 2048 fiber nodes, so the members take the symmetric kernel's partial sums and pull them together through the window,
with the cross kernel (and its pull of the periphery rows) off and on; the plan each shape takes is pinned.

The set-up contract of an empty block: a flow without fibers needs no fiber operators, no fiber preconditioner and no
links, for the partial operator (skb_flow_apply_matvec, skb_mflow_apply_matvec) too
(test_without_fibers_no_fiber_set_up_is_needed); a flow without periphery needs no dense handle; a flow without bodies
needs no body operators on one device, while a group member always calls skb_flow_group_set_body_operators (it lays
out the member's rows)."""
import contextlib

import numpy as np
import pytest

import skellysim_b200 as skb
import system_reference as sr
import system_rhs_reference as rr
from conftest import rel_l2, rel_max
from skellysim_b200 import capi, distributed
from test_gpu_flow import load
from test_gpu_group_system import Members, rhs_inputs, run_all
from test_gpu_system_matvec import make_case, setup_flow

pytestmark = pytest.mark.gpu
TOL = 1e-12
ETA, DT = 0.9, 1e-3

# single device: (fibers, periphery, bodies) with make_case's keywords
SINGLE = {"B": dict(n_fibers=0, n_shell=0, n_body_nodes=400, n_bodies=1),
          "BP": dict(n_fibers=0, n_shell=300, n_body_nodes=600, n_bodies=2),
          "F1": dict(n_fibers=1, n_shell=0, n_body_nodes=0, n_bodies=0, nodes=(32,)),
          "FP": dict(n_fibers=30, n_shell=300, n_body_nodes=0, n_bodies=0),
          "FB": dict(n_fibers=30, n_shell=0, n_body_nodes=600, n_bodies=2),
          "P": dict(n_fibers=0, n_shell=300, n_body_nodes=0, n_bodies=0),
          "Ffast": dict(n_fibers=150, n_shell=0, n_body_nodes=0, n_bodies=0, nodes=(32,)),
          "FPfast": dict(n_fibers=150, n_shell=500, n_body_nodes=0, n_bodies=0, nodes=(32,))}

# members of a group: the shape, the partition it must have on two and on three members (f0, f1, s0, s1, b0, b1), the
# plan the members take for their fiber rows (sym: the symmetric kernel's partial sums, pulled together through the
# window -- a member does so once the system has >= 2 x 1024 fiber nodes; otherwise its own rows with the plain
# kernel), and whether the RHS runs (it needs the class derivatives, which the device build has up to 128 nodes only)
MEMBERS = {
    # 2 fibers + 300 periphery + 2 bodies: on three members the middle one owns no fiber
    "M1": dict(kw=dict(n_fibers=2, n_shell=300, n_body_nodes=600, n_bodies=2), sym=False, rhs=True,
               parts={2: [(0, 1, 0, 150, 0, 300), (1, 2, 150, 300, 300, 600)],
                      3: [(0, 1, 0, 100, 0, 200), (1, 1, 100, 200, 200, 400), (1, 2, 200, 300, 400, 600)]}),
    # 30 fibers + 2 periphery nodes + 2 bodies: on three members the last one owns no periphery row
    "M2": dict(kw=dict(n_fibers=30, n_shell=2, n_body_nodes=600, n_bodies=2), sym=False, rhs=True,
               parts={2: [(0, 13, 0, 1, 0, 300), (13, 30, 1, 2, 300, 600)],
                      3: [(0, 8, 0, 1, 0, 200), (8, 21, 1, 2, 200, 400), (21, 30, 2, 2, 400, 600)]}),
    # fibers and periphery, no bodies: no link forces, no body rows in the window
    "M3": dict(kw=dict(n_fibers=30, n_shell=300, n_body_nodes=0, n_bodies=0), sym=False, rhs=True,
               parts={2: [(0, 13, 0, 150, 0, 0), (13, 30, 150, 300, 0, 0)],
                      3: [(0, 8, 0, 100, 0, 0), (8, 21, 100, 200, 0, 0), (21, 30, 200, 300, 0, 0)]}),
    # bodies only
    "M4": dict(kw=dict(n_fibers=0, n_shell=0, n_body_nodes=600, n_bodies=2), sym=False, rhs=True,
               parts={2: [(0, 0, 0, 0, 0, 300), (0, 0, 0, 0, 300, 600)],
                      3: [(0, 0, 0, 0, 0, 200), (0, 0, 0, 0, 200, 400), (0, 0, 0, 0, 400, 600)]}),
    # 2 periphery nodes and one body of 2 nodes: on three members the last one owns nothing at all
    "M5": dict(kw=dict(n_fibers=0, n_shell=2, n_body_nodes=2, n_bodies=1), sym=False, rhs=True,
               parts={2: [(0, 0, 0, 1, 0, 1), (0, 0, 1, 2, 1, 2)],
                      3: [(0, 0, 0, 1, 0, 1), (0, 0, 1, 2, 1, 2), (0, 0, 2, 2, 2, 2)]}),
    # M2 with 128-node fibers (3840 nodes): symmetric partials and, with the cross kernel, the pull of the periphery
    # rows -- of none on the last of three members
    "M2s": dict(kw=dict(n_fibers=30, n_shell=2, n_body_nodes=600, n_bodies=2, nodes=(128,)), sym=True, rhs=True,
                parts={2: [(0, 15, 0, 1, 0, 300), (15, 30, 1, 2, 300, 600)],
                       3: [(0, 10, 0, 1, 0, 200), (10, 20, 1, 2, 200, 400), (20, 30, 2, 2, 400, 600)]}),
    # M3 with 128-node fibers: symmetric partials and the cross kernel, no bodies
    "M3s": dict(kw=dict(n_fibers=30, n_shell=300, n_body_nodes=0, n_bodies=0, nodes=(128,)), sym=True, rhs=True,
                parts={2: [(0, 15, 0, 150, 0, 0), (15, 30, 150, 300, 0, 0)],
                       3: [(0, 10, 0, 100, 0, 0), (10, 20, 100, 200, 0, 0), (20, 30, 200, 300, 0, 0)]}),
    # two fibers of 1024 nodes and a periphery: on three members the first owns no fiber, yet takes its share of the
    # symmetric kernel's blocks, pulls no fiber row and its periphery rows' partials come from its peers
    # (its operators are 4096 x 4096 per fiber: the cross kernel on and three members only, where member 0 is empty)
    "M6s": dict(kw=dict(n_fibers=2, n_shell=300, n_body_nodes=0, n_bodies=0, nodes=(1024,)), sym=True, rhs=False,
                crosses=(1,), members=(1, 3),
                parts={2: [(0, 1, 0, 150, 0, 0), (1, 2, 150, 300, 0, 0)],
                       3: [(0, 0, 0, 100, 0, 0), (0, 1, 100, 200, 0, 0), (1, 2, 200, 300, 0, 0)]}),
}

MEMBER_SEED = 5  # make_case's seed of the member shapes: their node counts, and so the partition above
WORST = {}  # shape -> worst gate ratio (error / TOL) met


def edge_case(kw, seed, clamped=False, rhs=True):
    """make_case on the shape kw, with the RHS inputs of tests/test_gpu_group_system.py (the reference's class
    matrices, per-fiber parameters of all four boundary conditions, f_ext, F_T, point sources, a background flow);
    clamped: every fiber's minus end clamped.  rhs=False: no RHS (params and fparams None), and no class derivatives
    beyond the device build's 128 nodes"""
    fib, shell, bodies, ops, links, M, Minv, x = make_case(seed, **kw)
    shell = dict(shell, M=M, Minv=Minv)
    ops["A_inv"] = [np.linalg.inv(A) for A in ops["A"]]  # once (the set-up helpers take it)
    if not rhs:
        for d in ("D_2_0", "D_3_0", "D_4_0"):
            ops[d] = {n: m for n, m in ops[d].items() if n <= 128}
        src = rhs_inputs(dict(fib, n_nodes=[], lengths=[]), bodies, dict(ops, n_nodes=[]), seed)[2]
        return fib, shell, bodies, ops, links, x, None, None, src
    params, fparams, src = rhs_inputs(fib, bodies, ops, seed)
    if clamped:
        nfib = len(fib["n_nodes"])
        params = params[:5] + (np.ones(nfib, dtype=int),) + params[6:]
        for p in fparams:
            p["minus_clamped"] = True
    return fib, shell, bodies, ops, links, x, params, fparams, src


def references(fib, shell, bodies, ops, links, x, fparams, src):
    ns = shell["pos"].shape[0]
    mv = sr.system_apply_matvec(fib, shell, bodies, ops, links, shell["M"], x, ETA)[0]
    pc = sr.system_apply_preconditioner(ops["A"], ops["n_nodes"], shell["Minv"] if ns else None, bodies["A"],
                                        bodies["n_nodes"], x)
    rhs = None if fparams is None else rr.system_rhs(
        fib, shell, bodies, fparams, ETA, DT, f_ext=src["f_ext"], ft=src["ft"], points=src["points"],
        background=src["background"], v_growth=src["v_growth"], force_scale=src["force_scale"])[0]
    return mv, pc, rhs


def pieces(fib, shell, bodies):
    """(label, slice) of every block and of every body's node rows and six rows"""
    nf, ns = 4 * fib["pos"].shape[0], 3 * shell["pos"].shape[0]
    out = [("fibers", slice(0, nf)), ("shell", slice(nf, nf + ns))]
    off = nf + ns
    out.append(("bodies", slice(off, off + sum(3 * n + 6 for n in bodies["n_nodes"]))))
    for b, n in enumerate(bodies["n_nodes"]):
        out += [(f"body {b} nodes", slice(off, off + 3 * n)), (f"body {b} six", slice(off + 3 * n, off + 3 * n + 6))]
        off += 3 * n + 6
    return out


def gate(got, ref, fib, shell, bodies, shape, rhs=False):
    """every row finite; per piece max-norm and l2 at TOL (a RHS's six rows exactly +0.0); the worst ratio kept"""
    assert got.shape == ref.shape and np.isfinite(got).all(), (shape, np.flatnonzero(~np.isfinite(got))[:10])
    worst = 0.0
    for label, sl in pieces(fib, shell, bodies):
        g, r = got[sl], ref[sl]
        if rhs and label.endswith("six"):
            assert np.array_equal(g, np.zeros(6)) and not np.signbit(g).any(), (shape, label, g)
            continue
        if r.size == 0:
            continue
        e = max(rel_max(g, r), rel_l2(g, r))
        assert e <= TOL, (shape, label, e)
        worst = max(worst, e / TOL)
    WORST[shape] = max(WORST.get(shape, 0.0), worst)


def _nan(torch, n, dev):
    return torch.full((max(n, 1),), float("nan"), dtype=torch.float64, device=dev)


def single_device(fib, shell, bodies, ops, links, x, params, src, full_setup=True):
    """(matvec, preconditioner, RHS) of one flow, host and _device forms, each twice; the device outputs NaN first.
    full_setup=False: only the set-up a system's non-empty blocks need (no fiber operators, links or dense handle when
    their block is empty)."""
    import torch
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    ns, nb = shell["pos"].shape[0], len(bodies["n_nodes"])
    x0 = x.copy()
    with contextlib.ExitStack() as stack:
        fl = stack.enter_context(skb.Flow(0))
        dn = stack.enter_context(skb.Dense(device_ids=[0])) if ns else None
        if full_setup:
            setup_flow(fl, dn, fib, shell, bodies, ops, links)
        else:
            load(fl, fib, shell, dict(pos=bodies["pos"], normals=bodies["normals"], centers=bodies["centers"]))
            if nb:
                fl.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"],
                                      [np.linalg.inv(A) for A in bodies["A"]])
            if ns:
                dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, shell["M"])
                dn.set_matrix(skb.DENSE_M_INV, shell["Minv"])
        fl.set_point_sources(*src["points"])
        fl.set_background(*src["background"])
        assert fl.solution_size() == x.size
        kw = dict(v_growth=src["v_growth"], force_scale=src["force_scale"])
        host = {"mv": [fl.apply_system_matvec(x, ETA, dense=dn) for _ in range(2)],
                "pc": [fl.apply_system_preconditioner(x, dense=dn) for _ in range(2)],
                "rhs": [fl.build_system_rhs(*params, DT, ETA, f_external=src["f_ext"],
                                            body_forces_torques=src["ft"], **kw) for _ in range(2)]}
        d_x = t(x)
        d_f = t(src["f_ext"]) if fib["pos"].shape[0] else None
        d_F, d_T = (t(src["ft"][:, :3]), t(src["ft"][:, 3:])) if nb else (None, None)
        p = lambda a: a.data_ptr() if a is not None else 0
        device = {"mv": [], "pc": [], "rhs": []}
        for _ in range(2):
            outs = [_nan(torch, x.size, dev) for _ in range(3)]
            fl.apply_system_matvec_device(dn, d_x.data_ptr(), ETA, outs[0].data_ptr())
            fl.apply_system_preconditioner_device(dn, d_x.data_ptr(), outs[1].data_ptr())
            fl.build_system_rhs_device(*params, DT, ETA, p(d_f), p(d_F), p(d_T), outs[2].data_ptr(), **kw)
            torch.cuda.synchronize()
            for k, o in zip(("mv", "pc", "rhs"), outs):
                device[k].append(o[:x.size].cpu().numpy())
        assert np.array_equal(d_x.cpu().numpy(), x0)
    assert np.array_equal(x, x0)
    for k in host:
        for v in host[k] + device[k]:  # a row no launch wrote
            assert np.isfinite(v).all(), (k, np.flatnonzero(~np.isfinite(v))[:10])
        assert np.array_equal(host[k][0], host[k][1]), k             # reproducible
        assert np.array_equal(device[k][0], device[k][1]), k
        assert np.array_equal(device[k][0], host[k][0]), k           # the device form is the host form
    return host["mv"][0], host["pc"][0], host["rhs"][0]


@pytest.mark.parametrize("name", list(SINGLE))
def test_single_device_shapes_match_the_restatement(name):
    fib, shell, bodies, ops, links, x, params, fparams, src = edge_case(SINGLE[name], 91, clamped=name == "F1")
    ref_mv, ref_pc, ref_rhs = references(fib, shell, bodies, ops, links, x, fparams, src)
    mv, pc, rhs = single_device(fib, shell, bodies, ops, links, x, params, src)
    gate(mv, ref_mv, fib, shell, bodies, name)
    gate(pc, ref_pc, fib, shell, bodies, name)
    gate(rhs, ref_rhs, fib, shell, bodies, name, rhs=True)
    print(f"\n{name}: worst gate ratio {WORST[name]:.3f}")


@pytest.mark.parametrize("name", ["B", "BP", "P", "FP"])
def test_without_fibers_no_fiber_set_up_is_needed(name):
    """No fiber operators, preconditioner or links for a flow without fibers, no dense handle without a periphery:
    the same rows, bitwise, as with the empty uploads.  And a flow whose fibers all go away needs no new upload."""
    fib, shell, bodies, ops, links, x, params, fparams, src = edge_case(SINGLE[name], 92)
    full = single_device(fib, shell, bodies, ops, links, x, params, src)
    if fib["pos"].shape[0] == 0:
        bare = single_device(fib, shell, bodies, ops, links, x, params, src, full_setup=False)
        for a, b in zip(full, bare):
            assert np.array_equal(a, b)
        with skb.MultiFlow([0, 0]) as mf:  # two members, the same bare set-up
            mf.set_fibers(fib["pos"], [], [])
            mf.set_periphery(shell["pos"], shell["normals"])
            mf.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])
            if bodies["n_nodes"]:
                mf.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"],
                                      [np.linalg.inv(A) for A in bodies["A"]])
            if shell["pos"].shape[0]:
                mf.set_dense(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, shell["M"])
                mf.set_dense(skb.DENSE_M_INV, shell["Minv"])
            mf.set_point_sources(*src["points"])
            mf.set_background(*src["background"])
            got = (mf.apply_system_matvec(x, ETA), mf.apply_system_preconditioner(x),
                   mf.build_system_rhs(*params, DT, ETA, f_external=src["f_ext"], body_forces_torques=src["ft"],
                                       v_growth=src["v_growth"], force_scale=src["force_scale"]))
            _, apply_in, _ = partial_inputs(fib, shell, bodies, x, 96)
            m_partial = mf.apply_matvec(*apply_in, ETA)  # the partial operator takes no fiber set-up either
        for i, (g, o) in enumerate(zip(got, full)):
            gate(g, o, fib, shell, bodies, name, rhs=i == 2)
        ns = shell["pos"].shape[0]
        partial = []
        for bare in (False, True):
            with contextlib.ExitStack() as stack:
                fl = stack.enter_context(skb.Flow(0))
                dn = stack.enter_context(skb.Dense(device_ids=[0])) if ns else None
                if bare:
                    load(fl, fib, shell, dict(pos=bodies["pos"], normals=bodies["normals"], centers=bodies["centers"]))
                    if ns:
                        dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, shell["M"])
                else:
                    setup_flow(fl, dn, fib, shell, bodies, ops, links)
                partial.append(np.concatenate([np.ravel(a) for a in fl.apply_matvec(*apply_in, ETA, dense=dn)]))
        assert np.array_equal(partial[0], partial[1]) and np.isfinite(partial[1]).all()
        m_partial = np.concatenate([np.ravel(a) for a in m_partial])
        assert max(rel_max(m_partial, partial[0]), rel_l2(m_partial, partial[0])) <= TOL
        return
    # FP: fibers with their operators, then no fibers: the periphery alone, without another fiber upload
    no_fib = dict(pos=np.zeros((0, 3)), n_nodes=[], lengths=[])
    ps = edge_case(SINGLE["P"], 92)
    shell_p, src_p = ps[1], ps[8]
    rest = single_device(*ps[:7], src_p, full_setup=False)
    with skb.Flow(0) as fl, skb.Dense(device_ids=[0]) as dn:
        setup_flow(fl, dn, fib, shell, bodies, ops, links)
        fl.apply_system_matvec(x, ETA, dense=dn)
        load(fl, no_fib, shell_p, dict(pos=np.zeros((0, 3)), normals=np.zeros((0, 3)), centers=np.zeros((0, 3))))
        dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, shell_p["M"])
        dn.set_matrix(skb.DENSE_M_INV, shell_p["Minv"])
        fl.set_point_sources(*src_p["points"])
        fl.set_background(*src_p["background"])
        got = (fl.apply_system_matvec(ps[5], ETA, dense=dn), fl.apply_system_preconditioner(ps[5], dense=dn),
               fl.build_system_rhs(*ps[6], DT, ETA, f_external=src_p["f_ext"], body_forces_torques=src_p["ft"],
                                   v_growth=src_p["v_growth"], force_scale=src_p["force_scale"]))
    for a, b in zip(got, rest):
        assert np.array_equal(a, b)


def test_the_empty_system():
    """Nothing at all: a solution vector of length 0.  Every call succeeds, launches nothing and takes NULL vectors."""
    L = capi.library()
    empty = dict(pos=np.zeros((0, 3)), normals=np.zeros((0, 3)), centers=np.zeros((0, 3)))
    with skb.Flow(0) as fl:
        load(fl, dict(pos=np.zeros((0, 3)), n_nodes=[], lengths=[]), empty, empty)
        assert fl.solution_size() == 0
        calls = [lambda: L.skb_flow_apply_system_matvec(fl._h, None, None, ETA, None),
                 lambda: L.skb_flow_apply_system_matvec_device(fl._h, None, None, ETA, None, None),
                 lambda: L.skb_flow_apply_system_preconditioner(fl._h, None, None, None),
                 lambda: L.skb_flow_apply_system_preconditioner_device(fl._h, None, None, None, None),
                 lambda: L.skb_flow_build_system_rhs(fl._h, None, None, None, None, None, DT, ETA, None),
                 lambda: L.skb_flow_build_system_rhs_device(fl._h, None, None, None, None, None, None, DT, ETA, None,
                                                            None)]
        for call in calls:
            before = capi.launch_count()
            capi._check(call())
            assert capi.launch_count() == before
            assert fl.stats()["launches"] == 0
        assert fl.apply_system_matvec(np.zeros(0), ETA).size == 0
        assert fl.apply_system_preconditioner(np.zeros(0)).size == 0
        assert fl.build_system_rhs(1.0, 2.5e-3, 0.0125, 500.0, 1.0, 0, 0, DT, ETA).size == 0
    with skb.MultiFlow([0, 0]) as mf:
        mf.set_fibers(np.zeros((0, 3)), [], [])
        mf.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
        mf.set_bodies(np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3)))
        assert mf.apply_system_matvec(np.zeros(0), ETA).size == 0
        assert mf.apply_system_preconditioner(np.zeros(0)).size == 0
        assert mf.build_system_rhs(1.0, 2.5e-3, 0.0125, 500.0, 1.0, 0, 0, DT, ETA).size == 0


# ---- across members ----------------------------------------------------------------------------------------------

def mflow_device_lists():
    n = capi.device_count()
    return [[0], [0, 0], [0, 0, 0]] + [list(range(k)) for k in (2, 3) if n >= k]


def setup_mflow_edges(mf, fib, shell, bodies, ops, links):
    """tests/test_gpu_mflow_system.py's setup_mflow, each call also made for an empty block"""
    mf.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
    mf.set_periphery(shell["pos"], shell["normals"])
    mf.set_bodies(bodies["pos"], bodies["normals"], bodies["centers"])
    for n in ops["D_1_0"]:
        mf.set_fiber_class(n, ops["D_1_0"][n], ops["P"][n])
        if n in ops["D_2_0"]:
            mf.set_fiber_class_derivatives(n, ops["D_2_0"][n], ops["D_3_0"][n], ops["D_4_0"][n])
    mf.set_fiber_operators(ops["A"], ops["force"], ops["xs"], ops["length_prev"], ops["plus"])
    mf.set_fiber_preconditioner(ops["A_inv"])
    mf.set_body_operators(bodies["n_nodes"], bodies["weights"], bodies["ex"], bodies["ey"], bodies["ez"],
                          [np.linalg.inv(A) for A in bodies["A"]])
    mf.set_fiber_links(links["body"], links["site"], links["rigidity"])
    if shell["pos"].shape[0]:
        mf.set_dense(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, shell["M"])
        mf.set_dense(skb.DENSE_M_INV, shell["Minv"])


def partial_inputs(fib, shell, bodies, x, seed):
    rng = np.random.default_rng(seed)
    nf, ns, nb = fib["pos"].shape[0], shell["pos"].shape[0], bodies["pos"].shape[0]
    n_b = len(bodies["n_nodes"])
    strengths = (rng.uniform(-1, 1, (nf, 3)), rng.uniform(-1, 1, (ns, 3)), rng.uniform(-1, 1, (nb, 3)),
                 rng.uniform(-1, 1, (n_b, 6)))
    x_f, x_s = x[:4 * nf], x[4 * nf:4 * nf + 3 * ns].reshape(ns, 3)
    return strengths, (x_f, x_s, strengths[2], strengths[3]), rng.uniform(-2, 2, (50, 3))


def sequence(obj, x, params, src, rhs):
    """three consecutive matvecs, GMRES's interleaved P^-1, A, P^-1, A, the RHS twice"""
    mv = [obj.apply_system_matvec(x, ETA), obj.apply_system_matvec(x, ETA), obj.apply_system_matvec(2.0 * x, ETA)]
    seq = [obj.apply_system_preconditioner(x), obj.apply_system_matvec(x, ETA),
           obj.apply_system_preconditioner(2.0 * x), obj.apply_system_matvec(2.0 * x, ETA)]
    r = [rhs(obj), rhs(obj)] if rhs is not None else []
    return mv, seq, r


def cross_modes(shape):
    """the cross kernel off and on where the members take the symmetric plan (it needs that plan); auto elsewhere, where
    both would run the same code"""
    return shape.get("crosses", (0, 1) if shape["sym"] else (-1,))


class _One:
    """a single flow with the skb_mflow call signatures"""

    def __init__(self, fl, dn):
        self.fl, self.dn = fl, dn

    def apply_system_matvec(self, v, eta):
        return self.fl.apply_system_matvec(v, eta, dense=self.dn)

    def apply_system_preconditioner(self, v):
        return self.fl.apply_system_preconditioner(v, dense=self.dn)

    def build_system_rhs(self, *a, **k):
        return self.fl.build_system_rhs(*a, **k)


@pytest.mark.parametrize("name", list(MEMBERS))
def test_mflow_shapes_match_one_device_and_the_restatement(name):
    """Every skb_mflow call checks each member's group error after its launches and fails with SKB_ERR_STATE if a
    member met the flag time-out (mflow_collect_stats), so each call that returns is that check on every member."""
    shape = MEMBERS[name]
    fib, shell, bodies, ops, links, x, params, fparams, src = edge_case(shape["kw"], MEMBER_SEED, rhs=shape["rhs"])
    ref_mv, ref_pc, ref_rhs = references(fib, shell, bodies, ops, links, x, fparams, src)
    strengths, apply_in, r_trg = partial_inputs(fib, shell, bodies, x, 94)
    rhs_of = None
    if shape["rhs"]:
        rhs_kw = dict(f_external=src["f_ext"], body_forces_torques=src["ft"], v_growth=src["v_growth"],
                      force_scale=src["force_scale"])
        rhs_of = lambda o: o.build_system_rhs(*params, DT, ETA, **rhs_kw)
    ns = shell["pos"].shape[0]
    by_cross = {}
    for cross in cross_modes(shape):
        with contextlib.ExitStack() as stack:
            fl = stack.enter_context(skb.Flow(0))
            dn = stack.enter_context(skb.Dense(device_ids=[0])) if ns else None
            setup_flow(fl, dn, fib, shell, bodies, ops, links)
            fl.set_cross(cross)
            fl.set_point_sources(*src["points"])
            fl.set_background(*src["background"])
            one = sequence(_One(fl, dn), x, params, src, rhs_of)
            one_partial = (fl.matvec(*strengths, ETA), fl.apply_matvec(*apply_in, ETA, dense=dn),
                           fl.velocity_at_targets(r_trg, *strengths, ETA))
        for devs in (d for d in mflow_device_lists() if len(d) in shape.get("members", (1, 2, 3))):
            with skb.MultiFlow(devs) as mf:
                mf.set_cross(cross)
                setup_mflow_edges(mf, fib, shell, bodies, ops, links)
                mf.set_point_sources(*src["points"])
                mf.set_background(*src["background"])
                parts = [mf.partition(g) for g in range(len(devs))]
                if len(devs) in shape["parts"]:
                    assert parts == shape["parts"][len(devs)], (devs, parts)
                x0 = x.copy()
                got = sequence(mf, x, params, src, rhs_of)
                partial = (mf.matvec(*strengths, ETA), mf.apply_matvec(*apply_in, ETA),
                           mf.velocity_at_targets(r_trg, *strengths, ETA))
            assert np.array_equal(x, x0), devs
            mv, seq, rhs = got
            by_cross[cross, tuple(devs)] = mv[0]
            assert np.array_equal(mv[0], mv[1]) and np.array_equal(seq[1], mv[0]), devs
            assert np.array_equal(seq[3], mv[2]), devs
            for g, w in ((mv[0], ref_mv), (mv[2], 2.0 * ref_mv), (seq[0], ref_pc), (seq[2], 2.0 * ref_pc)):
                gate(g, w, fib, shell, bodies, name)
            if rhs:
                assert np.array_equal(rhs[0], rhs[1]), devs
                gate(rhs[0], ref_rhs, fib, shell, bodies, name, rhs=True)
            for i, (g, o) in enumerate(zip(mv + seq + rhs, one[0] + one[1] + one[2])):
                if len(devs) == 1:
                    assert np.array_equal(g, o), devs
                gate(g, o, fib, shell, bodies, name, rhs=i >= 7)
            for g, o in zip(partial, one_partial):
                g, o = (np.concatenate([np.ravel(a) for a in v]) if isinstance(v, tuple) else np.ravel(v)
                        for v in (g, o))
                assert np.isfinite(g).all(), devs
                if len(devs) == 1:
                    assert np.array_equal(g, o), devs
                if o.size:
                    assert max(rel_max(g, o), rel_l2(g, o)) <= TOL, devs
    if len(cross_modes(shape)) == 2 and ns >= 256:  # the cross kernel ran: the pairs are summed in another order
        for devs in ([0, 0], [0, 0, 0]):
            assert not np.array_equal(by_cross[0, tuple(devs)], by_cross[1, tuple(devs)]), devs
    print(f"\n{name}: worst gate ratio {WORST[name]:.3f}")


@pytest.mark.parametrize("name", list(MEMBERS))
def test_group_members_match_mflow_bitwise(name):
    """one thread per member, each on its own stream (tests/test_gpu_group_system.py); a member whose local vector is
    empty is accepted, through RankSystemOperator too.  The plan is pinned: with sym the members launch the symmetric
    kernel (skb_flow_last_sym_kernel), without it none does."""
    import torch
    shape = MEMBERS[name]
    fib, shell, bodies, ops, links, x, params, fparams, src = edge_case(shape["kw"], MEMBER_SEED, rhs=shape["rhs"])
    ref_mv, ref_pc, ref_rhs = references(fib, shell, bodies, ops, links, x, fparams, src)
    ns, fn = shell["pos"].shape[0], list(fib["n_nodes"])
    lists = [d for d in [[0, 0], [0, 0, 0]] + [list(range(k)) for k in (2, 3) if capi.device_count() >= k]
             if len(d) in shape.get("members", (2, 3))]
    for cross in cross_modes(shape):
        for devs in lists:
            with skb.MultiFlow(devs) as mf:
                mf.set_cross(cross)
                setup_mflow_edges(mf, fib, shell, bodies, ops, links)
                mf.set_point_sources(*src["points"])
                mf.set_background(*src["background"])
                m = [mf.apply_system_matvec(x, ETA), mf.apply_system_matvec(2.0 * x, ETA),
                     mf.apply_system_preconditioner(x)]
                if shape["rhs"]:
                    m.append(mf.build_system_rhs(*params, DT, ETA, f_external=src["f_ext"],
                                                 body_forces_torques=src["ft"], v_growth=src["v_growth"],
                                                 force_scale=src["force_scale"]))
            mem = Members(devs, fib, shell, bodies, ops, links, cross, src)
            try:
                assert [tuple(p) for p in mem.parts] == shape["parts"][len(devs)], (devs, mem.parts)
                assert np.array_equal(np.sort(np.concatenate(mem.rows)), np.arange(x.size))
                got = [mem.matvec(x), mem.matvec(2.0 * x), mem.matvec(x), mem.precondition(x),
                       mem.rhs(params, src) if shape["rhs"] else None,
                       mem.precondition(x), mem.matvec(x), mem.precondition(2.0 * x), mem.matvec(2.0 * x)]
                sym_pairs = [fl.last_sym_kernel()[1] for fl in mem.flows]
                assert (sum(sym_pairs) > 0) == shape["sym"], (devs, sym_pairs)
                # RankSystemOperator on the same members, the empty local vector included
                rso = [distributed.RankSystemOperator(fl, mem.dense[g], mem.dense[g], mem.parts[g], fn, ns,
                                                      bodies["n_nodes"], ETA, torch.device("cuda", devs[g]))
                       for g, fl in enumerate(mem.flows)]
                xl = [torch.from_numpy(np.ascontiguousarray(x[o.local_rows])).to(f"cuda:{d}")
                      for o, d in zip(rso, devs)]
                torch.cuda.synchronize()
                outs = {}

                def each(g):
                    with torch.cuda.stream(mem.streams[g]):
                        a = rso[g].apply(xl[g]).clone()
                        p = rso[g].apply_preconditioner(xl[g]).clone()
                    mem.streams[g].synchronize()
                    outs[g] = (a.cpu().numpy(), p.cpu().numpy())
                run_all(len(devs), each)
                assert mem.errors() == [-1] * len(devs), devs
            finally:
                mem.close()
            want = (m[0], m[1], m[0], m[2], m[3] if shape["rhs"] else None, m[2], m[0], None, m[1])
            for g, w in zip(got, want):
                if g is None:
                    continue
                assert np.isfinite(g).all(), devs
                if w is not None:
                    assert np.array_equal(g, w), devs
            for g, o in enumerate(rso):
                assert outs[g][0].size == o.local_rows.size
                assert np.array_equal(outs[g][0], m[0][o.local_rows])
                assert np.array_equal(outs[g][1], m[2][o.local_rows])
            gate(got[0], ref_mv, fib, shell, bodies, name)
            gate(got[3], ref_pc, fib, shell, bodies, name)
            if shape["rhs"]:
                gate(got[4], ref_rhs, fib, shell, bodies, name, rhs=True)
    print(f"\n{name}: worst gate ratio {WORST[name]:.3f}")


# ---- a closed form for the body block ----------------------------------------------------------------------------

def sphere(n, R):
    """n Fibonacci nodes on a sphere of radius R about the origin, their outward normals, equal weights 4 pi R^2 / n"""
    i = np.arange(n)
    z = 1.0 - (2 * i + 1) / n
    th = np.pi * (3.0 - np.sqrt(5.0)) * i
    s = np.sqrt(1.0 - z * z)
    e = np.stack([s * np.cos(th), s * np.sin(th), z], axis=1)
    return R * e, e, np.full(n, 4.0 * np.pi * R * R / n)


def host_body_solve(n, R, eta, F, L):
    """the discrete system of one sphere (shape B) on the host: A_ of body_operator, the RHS [-v(nodes); 0] of the
    centre Stokeslet and rotlet of F and L, a dense solve.  Returns (A, x)."""
    import oracle as orc
    r, nrm, w = sphere(n, R)
    ex, ey, ez = sr.singularity_vectors(r, nrm, w)
    A = sr.body_operator(r, nrm, np.zeros(3), w, ex, ey, ez)
    v = orc.body_flow(r, r, nrm, np.zeros_like(r), np.zeros((1, 3)), np.asarray(F)[None], np.asarray(L)[None], eta)
    return A, np.linalg.solve(A, np.concatenate([-v.reshape(-1), np.zeros(6)]))


def device_body_solve(n, R, eta, F, L, rtol):
    """the same system with A, P^-1 and the RHS from the device (SystemOperator), scipy GMRES on A P^-1"""
    import scipy.sparse.linalg as sla
    import torch
    from skellysim_b200.solver_hydro import SystemOperator
    r, nrm, w = sphere(n, R)
    ex, ey, ez = sr.singularity_vectors(r, nrm, w)
    A = sr.body_operator(r, nrm, np.zeros(3), w, ex, ey, ez)
    dev = torch.device("cuda", 0)
    to = lambda v: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).to(dev)
    with skb.Flow(0) as fl:  # a body alone: no fiber, periphery or link set-up
        fl.set_fibers(np.zeros((0, 3)), [], [])
        fl.set_periphery(np.zeros((0, 3)), np.zeros((0, 3)))
        fl.set_bodies(r, nrm, np.zeros((1, 3)))
        fl.set_body_operators([n], w, ex, ey, ez, [np.linalg.inv(A)])
        op = SystemOperator(fl, None, eta, dev)
        b = op.rhs((1.0, 2.5e-3, 0.0125, 500.0, 1.0, 0, 0), DT, body_forces=to(np.reshape(F, (1, 3))),
                   body_torques=to(np.reshape(L, (1, 3)))).cpu().numpy()
        Ad = lambda v: op.apply(to(v)).cpu().numpy()
        Pd = lambda v: op.apply_preconditioner(to(v)).cpu().numpy()
        N = op.n
        AP = sla.LinearOperator((N, N), matvec=lambda v: Ad(Pd(v)))
        z, info = sla.gmres(AP, b, rtol=rtol, atol=0.0, restart=200, maxiter=20)
        assert info == 0, info
        return Pd(z), b


def test_a_sphere_moves_by_stokes_law_and_turns_by_its_rotlet():
    """Shape B as a physical problem: a sphere of n = 400 Fibonacci nodes under a force F translates at F / (6 pi eta R)
    and under a torque L rotates at L / (8 pi eta R^3).  The device solve (scipy GMRES over A, P^-1 and the RHS of the
    device) is held to the host's dense solve of the same discrete system at rtol x cond(A), and to Stokes' law at twice
    the host's own discretisation error; the rotation, which this discretisation captures to rounding, to 1e-12 plus
    rtol."""
    n, rtol = 400, 1e-13
    R, eta, F = 1.0, 1.0, np.array([0.3, -0.7, 0.2])
    A, x_host = host_body_solve(n, R, eta, F, np.zeros(3))
    x_dev, _ = device_body_solve(n, R, eta, F, np.zeros(3), rtol)
    cond = np.linalg.cond(A)
    err_sys = np.linalg.norm(x_dev - x_host) / np.linalg.norm(x_host)
    assert err_sys <= 4 * rtol * cond, (err_sys, cond)
    U_stokes = F / (6 * np.pi * eta * R)
    e_host = np.linalg.norm(x_host[3 * n:3 * n + 3] - U_stokes) / np.linalg.norm(U_stokes)
    e_dev = np.linalg.norm(x_dev[3 * n:3 * n + 3] - U_stokes) / np.linalg.norm(U_stokes)
    assert e_dev <= 2 * e_host, (e_dev, e_host)
    R, eta, L = 0.5, 0.7, np.array([0.2, 0.5, -0.4])
    x_rot, _ = device_body_solve(n, R, eta, np.zeros(3), L, rtol)
    W = L / (8 * np.pi * eta * R ** 3)
    e_rot = np.linalg.norm(x_rot[3 * n + 3:] - W) / np.linalg.norm(W)
    assert e_rot <= 1e-12 + rtol, e_rot
    print(f"\nStokes drag, n = {n}: device {e_dev:.2e}, host {e_host:.2e}; |x_dev - x_host| / |x_host| {err_sys:.1e} "
          f"(cond {cond:.2f}); rotation {e_rot:.1e}")

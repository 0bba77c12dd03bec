"""GPU tests of skb_flow_build_fiber_operators (include/skelly_b200_flow.h): the per-fiber operators A_,
force_operator_, xs_ and A_^-1 built on the device from positions, lengths and per-fiber scalars, against the oracle's
statement-by-statement restatement of update_derivatives / update_linear_operator / apply_bc_rectangular /
update_force_operator (oracle/fiber_fd.py::FiberOperators) and numpy's inverse."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle as orc
import skellysim_b200 as skb
from oracle import fiber_fd
from conftest import rel_l2, rel_max
from test_gpu_flow import ft_of, load

pytestmark = pytest.mark.gpu
NODES = (8, 16, 24, 32, 48, 64, 96, 128)
ETA, DT = 0.9, 5e-3


def curved_fibers(seed, n_nodes):
    """Smooth curved fibers (an arc of a random helix per fiber), their lengths and random per-fiber scalars."""
    rng = np.random.default_rng(seed)
    pos, lengths = [], []
    for n in n_nodes:
        L = rng.uniform(0.6, 1.6)
        s = np.linspace(0.0, L, n)
        k, tau = rng.uniform(0.3, 1.5), rng.uniform(-1.0, 1.0)
        a = np.hypot(k, tau)                       # arc-length parametrised helix of curvature k, torsion tau
        c = np.stack([k / a ** 2 * np.cos(a * s), k / a ** 2 * np.sin(a * s), tau / a * s], axis=1)
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        pos.append(rng.uniform(-4, 4, 3) + c @ q.T)
        lengths.append(L)
    nf = len(n_nodes)
    combos = np.arange(nf) % 4                      # every (minus clamped, plus hinged) combination
    prm = dict(length_prev=np.array(lengths) * rng.uniform(0.95, 1.05, nf), bending_rigidity=rng.uniform(1e-3, 1e-2, nf),
               radius=rng.uniform(5e-3, 2e-2, nf), penalty_param=rng.uniform(100.0, 800.0, nf),
               beta_tstep=rng.uniform(0.5, 1.5, nf), minus_clamped=(combos & 1).astype(np.int32),
               plus_hinged=(combos >> 1).astype(np.int32))
    fib = dict(pos=np.concatenate(pos), n_nodes=[int(n) for n in n_nodes], lengths=lengths,
               forces=rng.uniform(-1, 1, (int(np.sum(n_nodes)), 3)))
    return fib, prm


def oracle_ops(fib, prm, f0=0, f1=None):
    f1 = len(fib["n_nodes"]) if f1 is None else f1
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
    fos = [fiber_fd.FiberOperators(fib["pos"][off[f]:off[f + 1]], fib["lengths"][f],
                                   bending_rigidity=prm["bending_rigidity"][f], radius=prm["radius"][f], eta=ETA,
                                   dt=DT, length_prev=prm["length_prev"][f], minus_clamped=bool(prm["minus_clamped"][f]),
                                   plus_pinned=bool(prm["plus_hinged"][f]), penalty_param=prm["penalty_param"][f],
                                   beta_tstep=prm["beta_tstep"][f]) for f in range(f0, f1)]
    ops = dict(n_nodes=[fo.n for fo in fos], A=[fo.A for fo in fos], force=[fo.force_operator for fo in fos],
               xs=np.concatenate([fo.xs for fo in fos]) if fos else np.zeros((0, 3)),
               length_prev=[fo.length_prev for fo in fos], plus=[fo.plus_bc_velocity for fo in fos], D_1_0={}, P={})
    for fo in fos:
        ops["D_1_0"][fo.n], ops["P"][fo.n] = fo.mats["D_1_0"], fo.mats["P_downsample_bc"]
    return ops


def set_classes(fl, n_nodes):
    for n in sorted(set(n_nodes)):
        m = fiber_fd.compute_matrices(n)
        fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
        fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])


def build(fl, prm, sl=slice(None)):
    fl.build_fiber_operators(*(prm[k][sl] for k in ("length_prev", "bending_rigidity", "radius", "penalty_param",
                                                    "beta_tstep", "minus_clamped", "plus_hinged")), DT, ETA)


def empty_shell_body(seed=0, n_shell=0, n_body=0):
    from test_gpu_flow import make_system
    _, shell, body = make_system(seed, 0, n_shell, n_body, 1 if n_body else 0)
    return shell, body


@pytest.fixture(scope="module")
def system():
    n_nodes = list(NODES) * 2
    np.random.default_rng(7).shuffle(n_nodes)
    fib, prm = curved_fibers(11, n_nodes)
    return fib, prm, oracle_ops(fib, prm)


def test_build_matches_oracle_operators_and_inverse(system):
    fib, prm, ops = system
    shell, body = empty_shell_body()
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])
        build(fl, prm)
        got = fl.get_fiber_operators()
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
    assert rel_max(got["xs"], ops["xs"]) <= 1e-12
    for f, n in enumerate(fib["n_nodes"]):
        A_ref = ops["A"][f]
        assert rel_max(got["A"][f], A_ref) <= 1e-12, (f, n, rel_max(got["A"][f], A_ref))
        assert rel_max(got["force"][f], ops["force"][f]) <= 1e-12, (f, n)
        assert rel_max(got["xs"][off[f]:off[f + 1]], ops["xs"][off[f]:off[f + 1]]) <= 1e-12, (f, n)
        X, X_np = got["A_inv"][f], np.linalg.inv(A_ref)
        cond = np.linalg.cond(A_ref)
        fwd = np.linalg.norm(X - X_np) / np.linalg.norm(X_np)
        assert fwd <= 1e-16 * cond, (f, n, fwd, cond)
        A = got["A"][f]
        res = np.linalg.norm(A @ X - np.eye(4 * n)) / (np.linalg.norm(A) * np.linalg.norm(X))
        assert res <= 1e-12, (f, n, res)


def test_apply_matvec_after_build(system):
    fib, prm, ops = system
    shell, body = empty_shell_body(3, 400, 120)
    rng = np.random.default_rng(5)
    nf, ns = fib["pos"].shape[0], shell["pos"].shape[0]
    x = rng.normal(size=4 * nf)
    link = rng.normal(size=(len(fib["n_nodes"]), 7))
    M = rng.normal(size=(3 * ns, 3 * ns)) / np.sqrt(3 * ns)
    with skb.Flow(0) as fl, skb.Dense(1) as dn:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])
        build(fl, prm)
        dn.set_matrix(skb.DENSE_STRESSLET_PLUS_COMPLEMENTARY, M)
        res, v_s, v_b = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
        res_d, res_shell, v_b_d = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link, dense=dn)
        y = fl.apply_fiber_preconditioner(x)
        got = fl.get_fiber_operators()
        # the same operators uploaded instead of built: bitwise the same matvec and preconditioner
        fl.set_fiber_operators(got["A"], got["force"], got["xs"], prm["length_prev"], prm["plus_hinged"])
        fl.set_fiber_preconditioner(got["A_inv"])
        res2, v_s2, v_b2 = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
        res2_d, _, _ = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link, dense=dn)
        y2 = fl.apply_fiber_preconditioner(x)
        # and a build after an upload replaces it again; two builds are bitwise equal
        build(fl, prm)
        again = fl.get_fiber_operators()
        res3, _, _ = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
    ref_res, ref_v = orc.apply_matvec_fibers(fib, shell, body, ops, x, ETA, link)
    for r in (res, res_d):
        assert rel_max(r, ref_res) <= 1e-12 and rel_l2(r, ref_res) <= 1e-12
    assert rel_max(v_s, ref_v[nf:nf + ns]) <= 1e-12 and rel_max(v_b, ref_v[nf + ns:]) <= 1e-12
    assert rel_max(res_shell.reshape(-1), orc.periphery_dense_apply(M, shell["density"].reshape(-1),
                                                                    v_s.reshape(-1))) <= 1e-12
    assert np.array_equal(res, res2) and np.array_equal(v_s, v_s2) and np.array_equal(v_b, v_b2)
    assert np.array_equal(res_d, res2_d) and np.array_equal(y, y2) and np.array_equal(res, res3)
    for k in ("A", "force", "A_inv"):
        assert all(np.array_equal(a, b) for a, b in zip(got[k], again[k]))
    assert np.array_equal(got["xs"], again["xs"])


@pytest.mark.parametrize("world", [2, 3])
def test_target_ranges_build_own_slice(system, world):
    from skellysim_b200.distributed import reference_rank_ranges
    fib, prm, _ = system
    shell, body = empty_shell_body(4, 90, 0)
    n_fibers, ns = len(fib["n_nodes"]), shell["pos"].shape[0]
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])
        build(fl, prm)
        full = fl.get_fiber_operators()
        off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
        for rank in range(world):
            f0, f1, s0, s1, b0, b1 = reference_rank_ranges(n_fibers, ns, 0, rank, world)
            fl.set_target_ranges(f0, f1, s0, s1, b0, b1)
            build(fl, prm, slice(f0, f1))
            own = fl.get_fiber_operators()
            for k in ("A", "force", "A_inv"):
                assert len(own[k]) == f1 - f0
                assert all(np.array_equal(a, b) for a, b in zip(own[k], full[k][f0:f1]))
            assert np.array_equal(own["xs"], full["xs"][off[f0]:off[f1]])


def test_multiflow_build(system):
    fib, prm, _ = system
    shell, body = empty_shell_body(5, 300, 0)
    rng = np.random.default_rng(6)
    nf = fib["pos"].shape[0]
    x = rng.normal(size=4 * nf)
    link = rng.normal(size=(len(fib["n_nodes"]), 7))
    args = [prm[k] for k in ("length_prev", "bending_rigidity", "radius", "penalty_param", "beta_tstep",
                             "minus_clamped", "plus_hinged")]
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])
        build(fl, prm)
        ref = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
    for devices in ([0, 0], [0, 0, 0]):
        with skb.MultiFlow(devices) as mf:
            mf.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
            mf.set_periphery(shell["pos"], shell["normals"])
            mf.set_bodies(body["pos"], body["normals"], body["centers"])
            for n in sorted(set(fib["n_nodes"])):
                m = fiber_fd.compute_matrices(n)
                mf.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
                mf.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
            mf.build_fiber_operators(*args, DT, ETA)
            res, o_s, v_b = mf.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
        assert rel_max(res, ref[0]) <= 1e-12 and rel_max(o_s, ref[1]) <= 1e-12, devices


def test_build_rejections():
    fib, prm = curved_fibers(12, [8, 16, 16])
    shell, body = empty_shell_body()
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        m8, m16 = fiber_fd.compute_matrices(8), fiber_fd.compute_matrices(16)
        fl.set_fiber_class(8, m8["D_1_0"], m8["P_downsample_bc"])
        fl.set_fiber_class_derivatives(8, m8["D_2_0"], m8["D_3_0"], m8["D_4_0"])
        with pytest.raises(skb.SkbError, match=r"fiber 1 has 16 nodes but skb_flow_set_fiber_class\("):
            build(fl, prm)
        fl.set_fiber_class(16, m16["D_1_0"], m16["P_downsample_bc"])
        with pytest.raises(skb.SkbError, match=r"fiber 1 has 16 nodes but skb_flow_set_fiber_class_derivatives"):
            build(fl, prm)
        fl.set_fiber_class_derivatives(16, m16["D_2_0"], m16["D_3_0"], m16["D_4_0"])
        build(fl, prm)
        for key, bad, pat in (("length_prev", 0.0, "fiber 2: length_prev"), ("radius", -1.0, "fiber 2: .*radius"),
                              ("minus_clamped", 2, "fiber 2: minus_clamped = 2"),
                              ("plus_hinged", -1, "fiber 2: .*plus_hinged = -1")):
            p = {k: np.array(v) for k, v in prm.items()}
            p[key][2] = bad
            with pytest.raises(skb.SkbError, match=pat):
                build(fl, p)
        with pytest.raises(skb.SkbError, match="dt = 0"):
            fl.build_fiber_operators(1.0, 1e-3, 1e-2, 500.0, 1.0, 0, 0, 0.0, ETA)
        with pytest.raises(skb.SkbError, match="eta = -1"):
            fl.build_fiber_operators(1.0, 1e-3, 1e-2, 500.0, 1.0, 0, 0, DT, -1.0)
        # a refused build leaves no operators behind
        with pytest.raises(skb.SkbError, match="set_fiber_operators"):
            fl.apply_fiber_force(np.zeros(4 * fib["pos"].shape[0]))
        with pytest.raises(skb.SkbError, match="8 <= n <= 128"):
            fl.set_fiber_class_derivatives(7, np.zeros((7, 7)), np.zeros((7, 7)), np.zeros((7, 7)))
    fib7, prm7 = curved_fibers(13, [7])
    with skb.Flow(0) as fl:
        load(fl, fib7, shell, body)
        fl.set_fiber_class(7, np.eye(7), np.zeros((14, 28)))  # (no 8-point stencil exists on 7 nodes)
        with pytest.raises(skb.SkbError, match="fiber 0 has 7 nodes: the device build takes 8 <= n <= 128"):
            build(fl, prm7)


def test_cpp_mirror_build(tmp_path):
    # tests/cpp/fiber_build_test.cpp: flow.hpp build -> read back -> upload round trip -> identical matvec; compiled here
    # against the in-tree headers and library
    here = os.path.dirname(os.path.abspath(__file__))
    root, libdir = os.path.dirname(here), os.path.dirname(skb.library_path())
    cxx = shutil.which("g++") or shutil.which("c++")
    assert cxx, "a C++ compiler is needed to build tests/cpp/fiber_build_test.cpp"
    exe = str(tmp_path / "fiber_build_test")
    subprocess.run([cxx, "-O2", "-std=c++17", "-Wall", "-I", os.path.join(root, "include"), "-o", exe,
                    os.path.join(here, "cpp", "fiber_build_test.cpp"), "-L", libdir, "-lskelly_b200",
                    f"-Wl,-rpath,{libdir}"], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr

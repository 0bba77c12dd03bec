"""GPU tests of skb_flow_build_fiber_rhs (include/skelly_b200_flow.h): the fiber block of the RHS formed on the device.

The RHS is held entry by entry to |dev - ext| <= C_RHS u S against the long-double reference
(fiber_rhs_reference.fiber_rhs; tests/test_fiber_rhs_cpu.py shows the criterion attainable and sharp): curved fibers
with n = 8 .. 128 mixed in
one container, all four boundary-condition combinations, with and without each optional input, in the host form and
the device form on a non-default stream.  Also: a straight free fiber in a uniform flow is advected through the device
operators and their inverse; target ranges and MultiFlow tile the single-flow result bitwise; an RHS call leaves the
resident operators, their inverse and the matvec bitwise unchanged; class matrices replaced after use, or set in
another order of n, leave the build, the RHS and the matvec bitwise as a flow that only saw the final ones; every
rejection comes before any launch."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import skellysim_b200 as skb
from skellysim_b200 import capi
from fiber_rhs_reference import fiber_rhs
from test_fiber_rhs_cpu import C_RHS, advection_case, ratio
from test_gpu_fiber_build import (DT, ETA, NODES, build, curved_fibers, empty_shell_body, fiber_operators,
                                  set_classes)
from test_gpu_flow import ft_of, load

PARAMS = ("length_prev", "bending_rigidity", "radius", "penalty_param", "beta_tstep", "minus_clamped", "plus_hinged")
VARIANTS = ("all", "no_v", "no_f", "no_growth", "no_motor", "none")


def inputs(fib, seed=3):
    rng = np.random.default_rng(seed)
    nf, nfib = fib["pos"].shape[0], len(fib["n_nodes"])
    return dict(v_on_fibers=rng.uniform(-1, 1, (nf, 3)), f_external=rng.uniform(-1, 1, (nf, 3)),
                v_growth=rng.uniform(-1, 1, nfib), force_scale=rng.uniform(-2, 2, nfib))


def variant(inp, name):
    drop = dict(all=(), no_v=("v_on_fibers",), no_f=("f_external",), no_growth=("v_growth",),
                no_motor=("force_scale",), none=tuple(inp))[name]
    return {k: (None if k in drop else v) for k, v in inp.items()}


def rhs_host(fl, prm, inp, sl=slice(None), dt=DT):
    return fl.build_fiber_rhs(*(prm[k][sl] for k in PARAMS), dt, ETA, **inp)


def extended_rhs(fib, prm, inp):
    """per fiber: (ext, S) of every variant"""
    ext, S = fiber_operators(fib, prm, DT, dtype=np.longdouble), fiber_operators(fib, prm, DT, absolute=True)
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
    out = {}
    for name in VARIANTS:
        d = variant(inp, name)
        per = []
        for f, (e, s) in enumerate(zip(ext, S)):
            sl = slice(off[f], off[f + 1])
            kw = dict(v=None if d["v_on_fibers"] is None else d["v_on_fibers"][sl],
                      f_external=None if d["f_external"] is None else d["f_external"][sl],
                      force_scale=None if d["force_scale"] is None else d["force_scale"][f],
                      v_growth=0.0 if d["v_growth"] is None else d["v_growth"][f])
            per.append((fiber_rhs(e, **kw), fiber_rhs(s, **kw)))
        out[name] = per
    return out


def check_rhs(got, fib, ref, label):
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
    worst = 0.0
    for f, (ext, S) in enumerate(ref):
        r = ratio(got[4 * off[f]:4 * off[f + 1]], ext, S)
        assert r <= C_RHS, (label, f, fib["n_nodes"][f], r)
        worst = max(worst, r)
    return worst


@pytest.fixture(scope="module")
def system():
    n_nodes = list(NODES) * 2
    np.random.default_rng(17).shuffle(n_nodes)
    fib, prm = curved_fibers(19, n_nodes)
    inp = inputs(fib)
    return fib, prm, inp, extended_rhs(fib, prm, inp)


@pytest.mark.gpu
def test_rhs_matches_extended_oracle(system):
    fib, prm, inp, ref = system
    shell, body = empty_shell_body()
    worst = {}
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])                  # no operators: the RHS does not need them
        for name in VARIANTS:
            got = rhs_host(fl, prm, variant(inp, name))
            worst[name] = check_rhs(got, fib, ref[name], name)
            st = fl.stats()
            assert st["launches"] == 1 and st["device_ms"] > 0 and st["total_ms"] >= st["device_ms"]
    print("\ndevice RHS |d|/(u S), worst per variant:", {k: round(v, 2) for k, v in worst.items()})


@pytest.mark.gpu
def test_device_form_on_a_side_stream(system):
    torch = pytest.importorskip("torch")
    fib, prm, inp, ref = system
    shell, body = empty_shell_body()
    dev = torch.device("cuda:0")
    nf = fib["pos"].shape[0]
    side = torch.cuda.Stream(device=dev)
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])
        for name in ("all", "no_v", "no_f", "none"):
            d = variant(inp, name)
            host = rhs_host(fl, prm, d)
            with torch.cuda.stream(side):
                t = {k: None if d[k] is None else torch.from_numpy(d[k]).to(dev)
                     for k in ("v_on_fibers", "f_external")}
                d_rhs = torch.full((4 * nf,), np.nan, dtype=torch.float64, device=dev)
                fl.build_fiber_rhs_device(*(prm[k] for k in PARAMS), DT, ETA,
                                          0 if t["v_on_fibers"] is None else t["v_on_fibers"].data_ptr(),
                                          0 if t["f_external"] is None else t["f_external"].data_ptr(),
                                          d_rhs.data_ptr(), v_growth=d["v_growth"], force_scale=d["force_scale"],
                                          stream=side.cuda_stream)
                got = d_rhs.cpu().numpy()                 # (ordered on the side stream)
            assert fl.stats()["launches"] == 1
            assert np.array_equal(got, host), name
            check_rhs(got, fib, ref[name], "device " + name)


@pytest.mark.gpu
def test_straight_fiber_is_advected_through_the_device_inverse():
    dt = 5e-3
    n_nodes = list(NODES)
    pos, lengths, U = [], [], []
    for n in n_nodes:
        x, L, Uf = advection_case(n, seed=7)
        pos.append(x)
        lengths.append(L)
        U.append(np.tile(Uf, (n, 1)))
    fib = dict(pos=np.concatenate(pos), n_nodes=n_nodes, lengths=lengths)
    nfib = len(n_nodes)
    prm = dict(length_prev=np.array(lengths), bending_rigidity=np.full(nfib, 2.5e-3), radius=np.full(nfib, 0.0125),
               penalty_param=np.full(nfib, 500.0), beta_tstep=np.ones(nfib), minus_clamped=np.zeros(nfib, np.int32),
               plus_hinged=np.zeros(nfib, np.int32))
    shell, body = empty_shell_body()
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_classes(fl, n_nodes)
        build(fl, prm, dt=dt)
        rhs = rhs_host(fl, prm, dict(v_on_fibers=np.concatenate(U)), dt=dt)
        y = fl.apply_fiber_preconditioner(rhs)
        A = fl.get_fiber_operators(inverse=False)["A"]
    off = np.concatenate([[0], np.cumsum(n_nodes)])
    for f, n in enumerate(n_nodes):
        sl = slice(4 * off[f], 4 * off[f + 1])
        want = np.concatenate([(pos[f] + dt * U[f]).T.reshape(-1), np.zeros(n)])
        y_np = np.linalg.solve(A[f], rhs[sl])
        for part in (slice(0, 3 * n), slice(3 * n, 4 * n)):
            e_dev = np.abs(y[sl][part] - want[part]).max()
            e_np = np.abs(y_np[part] - want[part]).max()
            assert e_dev <= 32 * e_np + 1e-14, (n, part, e_dev, e_np)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_target_ranges_tile_the_whole_container(system, world):
    from skellysim_b200.distributed import reference_rank_ranges
    fib, prm, inp, _ = system
    shell, body = empty_shell_body(4, 90, 0)
    n_fibers, ns = len(fib["n_nodes"]), shell["pos"].shape[0]
    off = np.concatenate([[0], np.cumsum(fib["n_nodes"])])
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])
        full = rhs_host(fl, prm, inp)
        for rank in range(world):
            f0, f1, s0, s1, b0, b1 = reference_rank_ranges(n_fibers, ns, 0, rank, world)
            fl.set_target_ranges(f0, f1, s0, s1, b0, b1)
            own = {k: None if v is None else v[off[f0]:off[f1]] if v.ndim == 2 else v[f0:f1] for k, v in inp.items()}
            got = rhs_host(fl, prm, own, slice(f0, f1))
            assert np.array_equal(got, full[4 * off[f0]:4 * off[f1]]), (world, rank)


@pytest.mark.gpu
def test_multiflow_rhs(system):
    fib, prm, inp, _ = system
    shell, body = empty_shell_body(5, 300, 0)
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])
        ref = rhs_host(fl, prm, inp)
    for devices in ([0, 0], [0, 0, 0]):
        with skb.MultiFlow(devices) as mf:
            mf.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
            mf.set_periphery(shell["pos"], shell["normals"])
            mf.set_bodies(body["pos"], body["normals"], body["centers"])
            set_classes(mf, fib["n_nodes"])
            got = mf.build_fiber_rhs(*(prm[k] for k in PARAMS), DT, ETA, **inp)
        assert np.array_equal(got, ref), devices


@pytest.mark.gpu
def test_rhs_leaves_the_operators_untouched(system):
    fib, prm, inp, _ = system
    shell, body = empty_shell_body(3, 200, 60)
    rng = np.random.default_rng(5)
    nf = fib["pos"].shape[0]
    x = rng.normal(size=4 * nf)
    link = rng.normal(size=(len(fib["n_nodes"]), 7))

    def matvec(fl):
        res = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
        return res + (fl.apply_fiber_preconditioner(x),)

    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_classes(fl, fib["n_nodes"])
        for how in ("built", "uploaded"):
            if how == "built":
                build(fl, prm)
            else:
                ops = fl.get_fiber_operators()
                fl.set_fiber_operators(ops["A"], ops["force"], ops["xs"], prm["length_prev"], prm["plus_hinged"])
                fl.set_fiber_preconditioner(ops["A_inv"])
            before, ops0 = matvec(fl), fl.get_fiber_operators()
            first = rhs_host(fl, prm, inp)
            # class derivatives set again (same values, the operators stay): the class table is uploaded anew under
            # the resident operators, whose GEMV reads it at the same offsets
            n = fib["n_nodes"][0]
            m = fiber_fd_matrices(n)
            fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
            assert np.array_equal(rhs_host(fl, prm, inp), first), how
            after, ops1 = matvec(fl), fl.get_fiber_operators()
            for a, b in zip(before, after):
                assert np.array_equal(a, b), how
            for k in ("A", "force", "A_inv"):
                assert all(np.array_equal(a, b) for a, b in zip(ops0[k], ops1[k])), (how, k)
            assert np.array_equal(ops0["xs"], ops1["xs"]), how


def set_class_matrices(fl, n_values, scale=1.0, derivatives_first=False):
    for n in n_values:
        m = {k: v * scale for k, v in fiber_fd_matrices(n).items() if k.startswith(("D_", "P_downsample"))}
        calls = [lambda: fl.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"]),
                 lambda: fl.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])]
        for call in calls[::-1] if derivatives_first else calls:
            call()


def class_table_outputs(fl, fib, prm, inp, shell, body):
    """what the class table feeds: the build's operators and inverse, the RHS, the matvec and the preconditioner"""
    rng = np.random.default_rng(5)
    x = rng.normal(size=4 * fib["pos"].shape[0])
    link = rng.normal(size=(len(fib["n_nodes"]), 7))
    return (fl.get_fiber_operators(), rhs_host(fl, prm, inp),
            fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link) +
            (fl.apply_fiber_preconditioner(x),))


def assert_same_outputs(got, want, label):
    ops, rhs, mv = got
    for k in ("A", "force", "A_inv"):
        assert all(np.array_equal(a, b) for a, b in zip(ops[k], want[0][k])), (label, k)
    assert np.array_equal(ops["xs"], want[0]["xs"]), label
    assert np.array_equal(rhs, want[1]), label
    for a, b in zip(mv, want[2]):
        assert np.array_equal(a, b), label


@pytest.mark.gpu
@pytest.mark.parametrize("derivatives_first", [False, True])
def test_class_matrices_replaced(system, derivatives_first):
    """perturbed class matrices in use (a build, an RHS, uploaded operators), then the real ones again: every output
    equals a flow's that only ever saw the real ones"""
    fib, prm, inp, _ = system
    shell, body = empty_shell_body(3, 200, 60)
    n_values = sorted(set(fib["n_nodes"]))
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_class_matrices(fl, n_values)
        build(fl, prm)
        want = class_table_outputs(fl, fib, prm, inp, shell, body)
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        set_class_matrices(fl, n_values, scale=1.0 + 1e-3)
        build(fl, prm)
        perturbed = rhs_host(fl, prm, inp)
        assert not np.array_equal(perturbed, want[1])
        ops = fl.get_fiber_operators()
        fl.set_fiber_operators(ops["A"], ops["force"], ops["xs"], prm["length_prev"], prm["plus_hinged"])
        fl.set_fiber_preconditioner(ops["A_inv"])
        set_class_matrices(fl, n_values, derivatives_first=derivatives_first)
        build(fl, prm)
        assert_same_outputs(class_table_outputs(fl, fib, prm, inp, shell, body), want, derivatives_first)


@pytest.mark.gpu
def test_class_order_does_not_matter(system):
    """the classes set in ascending and in descending n give the same operators, RHS and matvec"""
    fib, prm, inp, _ = system
    shell, body = empty_shell_body(3, 200, 60)
    out = []
    for n_values in (sorted(set(fib["n_nodes"])), sorted(set(fib["n_nodes"]), reverse=True)):
        with skb.Flow(0) as fl:
            load(fl, fib, shell, body)
            set_class_matrices(fl, n_values)
            build(fl, prm)
            out.append(class_table_outputs(fl, fib, prm, inp, shell, body))
    assert_same_outputs(out[1], out[0], "descending")


@pytest.mark.gpu
def test_rhs_rejections():
    fib, prm = curved_fibers(12, [8, 16, 16])
    shell, body = empty_shell_body()
    inp = inputs(fib)
    L = capi.library()
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        m8, m16 = fiber_fd_matrices(8), fiber_fd_matrices(16)
        fl.set_fiber_class(8, m8["D_1_0"], m8["P_downsample_bc"])
        fl.set_fiber_class_derivatives(8, m8["D_2_0"], m8["D_3_0"], m8["D_4_0"])

        def refused(pat, call):
            before = capi.launch_count()
            with pytest.raises(skb.SkbError, match=pat) as e:
                call()
            assert "error 1:" in str(e.value)                       # SKB_ERR_INVALID
            assert capi.launch_count() == before, pat

        refused(r"fiber 1 has 16 nodes but skb_flow_set_fiber_class\(", lambda: rhs_host(fl, prm, inp))
        fl.set_fiber_class(16, m16["D_1_0"], m16["P_downsample_bc"])
        refused("fiber 1 has 16 nodes but skb_flow_set_fiber_class_derivatives", lambda: rhs_host(fl, prm, inp))
        fl.set_fiber_class_derivatives(16, m16["D_2_0"], m16["D_3_0"], m16["D_4_0"])
        good = rhs_host(fl, prm, inp)
        for key, bad, pat in (("length_prev", 0.0, "fiber 2: length_prev"), ("radius", -1.0, "fiber 2: .*radius"),
                              ("minus_clamped", 2, "fiber 2: minus_clamped = 2"),
                              ("plus_hinged", -1, "fiber 2: .*plus_hinged = -1")):
            p = {k: np.array(v) for k, v in prm.items()}
            p[key][2] = bad
            refused(pat, lambda: rhs_host(fl, p, inp))
        for key, bad, pat in (("v_growth", np.nan, "fiber 1: v_growth = nan"),
                              ("force_scale", np.inf, "fiber 0: .*force_scale = inf")):
            d = dict(inp)
            d[key] = np.array(inp[key])
            d[key][0 if key == "force_scale" else 1] = bad
            refused(pat, lambda: rhs_host(fl, prm, d))
        refused("dt = 0", lambda: rhs_host(fl, prm, inp, dt=0.0))
        refused("eta = -1", lambda: fl.build_fiber_rhs(*(prm[k] for k in PARAMS), DT, -1.0))
        p = capi.fiber_params(3, *(prm[k] for k in PARAMS))
        out = np.zeros(4 * fib["pos"].shape[0])
        for args in ((None, capi._p(out)), (capi._params_ptr(p), None)):
            before = capi.launch_count()
            assert L.skb_flow_build_fiber_rhs(fl._h, args[0], None, None, None, None, DT, ETA, args[1]) == 1
            assert b"NULL argument" in L.skb_last_error_string() and capi.launch_count() == before
        assert np.array_equal(rhs_host(fl, prm, inp), good)         # nothing was left half done
    fib7, prm7 = curved_fibers(13, [7])
    with skb.Flow(0) as fl:
        load(fl, fib7, shell, body)
        fl.set_fiber_class(7, np.eye(7), np.zeros((14, 28)))
        with pytest.raises(skb.SkbError, match="fiber 0 has 7 nodes: the device build takes 8 <= n <= 128"):
            rhs_host(fl, prm7, {})


def fiber_fd_matrices(n):
    from oracle import fiber_fd
    return fiber_fd.compute_matrices(n)


@pytest.mark.gpu
def test_cpp_mirror_rhs(tmp_path):
    # tests/cpp/fiber_rhs_test.cpp: flow.hpp build_fiber_rhs against the C ABI; compiled here against the in-tree
    # headers and library
    here = os.path.dirname(os.path.abspath(__file__))
    root, libdir = os.path.dirname(here), os.path.dirname(skb.library_path())
    cxx = shutil.which("g++") or shutil.which("c++")
    assert cxx, "a C++ compiler is needed to build tests/cpp/fiber_rhs_test.cpp"
    exe = str(tmp_path / "fiber_rhs_test")
    subprocess.run([cxx, "-O2", "-std=c++17", "-Wall", "-I", os.path.join(root, "include"), "-o", exe,
                    os.path.join(here, "cpp", "fiber_rhs_test.cpp"), "-L", libdir, "-lskelly_b200",
                    f"-Wl,-rpath,{libdir}"], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr

"""GPU test of the handles' create and destroy paths: a create that fails part-way releases what it had built (the
destructors run on half-built objects), and repeated create / destroy cycles leave the library computing correctly.
Leaks are not measured here: every device resource has one owner that releases it (test_capi_exports.py checks the
sources for releases outside those owners)."""
import ctypes as C

import numpy as np
import pytest

import oracle as orc
import skellysim_b200 as skb
from conftest import rel_max
from oracle import fiber_fd
from skellysim_b200 import capi
from test_gpu_fiber_build import DT, ETA, build, curved_fibers, empty_shell_body, oracle_ops, set_classes
from test_gpu_flow import ft_of, load

pytestmark = pytest.mark.gpu
SKB_ERR_INVALID = 1  # include/skelly_b200.h


def test_failed_ctx_and_dense_creates_unwind():
    # two ids pass the device-count check only with two devices visible; then device 0 is set up before the
    # out-of-range second id is refused
    if capi.device_count() < 2:
        pytest.skip("needs 2 GPUs: with one, n_gpus = 2 is refused before any device is set up")
    L = capi.library()
    ids = (C.c_int * 2)(0, 99)
    for create in (L.skb_ctx_create_on, L.skb_dense_create_on):
        for _ in range(50):
            h = C.c_void_p()
            assert create(ids, 2, C.byref(h)) == SKB_ERR_INVALID
            assert b"device id 99 out of range" in L.skb_last_error_string()
            assert not h.value


def test_failed_multiflow_create_unwinds():
    # member 0's flow (6 contexts, stream, events) and its I/O events exist when member 1's device is refused
    for _ in range(5):
        with pytest.raises(skb.SkbError, match="device 99 out of range"):
            skb.MultiFlow([0, 99])


def test_create_destroy_cycles_keep_results():
    fib, prm = curved_fibers(21, [8, 16, 32, 64] * 2)
    ops = oracle_ops(fib, prm)
    shell, body = empty_shell_body(6, 200, 60)
    rng = np.random.default_rng(8)
    nf = fib["pos"].shape[0]
    x = rng.normal(size=4 * nf)
    link = rng.normal(size=(len(fib["n_nodes"]), 7))
    ref_res, ref_v = orc.apply_matvec_fibers(fib, shell, body, ops, x, ETA, link)
    args = [prm[k] for k in ("length_prev", "bending_rigidity", "radius", "penalty_param", "beta_tstep",
                             "minus_clamped", "plus_hinged")]
    ns = shell["pos"].shape[0]
    first = None
    for _ in range(5):
        with skb.Flow(0) as fl:
            load(fl, fib, shell, body)
            set_classes(fl, fib["n_nodes"])
            build(fl, prm)
            res, v_s, v_b = fl.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
        assert rel_max(res, ref_res) <= 1e-12
        assert rel_max(v_s, ref_v[nf:nf + ns]) <= 1e-12 and rel_max(v_b, ref_v[nf + ns:]) <= 1e-12
        if first is None:
            first = res
        assert np.array_equal(res, first)
        with skb.MultiFlow([0, 0]) as mf:
            mf.set_fibers(fib["pos"], fib["n_nodes"], fib["lengths"])
            mf.set_periphery(shell["pos"], shell["normals"])
            mf.set_bodies(body["pos"], body["normals"], body["centers"])
            for n in sorted(set(fib["n_nodes"])):
                m = fiber_fd.compute_matrices(n)
                mf.set_fiber_class(n, m["D_1_0"], m["P_downsample_bc"])
                mf.set_fiber_class_derivatives(n, m["D_2_0"], m["D_3_0"], m["D_4_0"])
            mf.build_fiber_operators(*args, DT, ETA)
            res_m, v_s_m, v_b_m = mf.apply_matvec(x, shell["density"], body["density"], ft_of(body), ETA, link)
        assert rel_max(res_m, res) <= 1e-12 and rel_max(v_s_m, v_s) <= 1e-12 and rel_max(v_b_m, v_b) <= 1e-12

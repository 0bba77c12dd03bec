"""CPU tests of the drop-in boundary: the C-ABI library loads, exports every symbol include/*.h declares and
the reference-named C++ symbols, and refuses (loudly, with an error code) to compute without a GPU."""
import ctypes as C
import glob
import os
import re

import numpy as np
import pytest

import skellysim_b200 as skb
from skellysim_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    names = []
    for h in glob.glob(os.path.join(ROOT, "include", "*.h")):
        src = open(h).read()
        names += re.findall(r"SKB_API\s+[\w\s\*]+?\b(skb_\w+)\s*\(", src)
    return sorted(set(names))


def test_header_declares_something():
    names = _declared_functions()
    assert "skb_eval" in names and "skb_stokeslet_direct" in names and len(names) >= 20


def test_library_exports_every_declared_symbol():
    L = C.CDLL(skb.library_path())
    missing = [n for n in _declared_functions() if not hasattr(L, n)]
    assert not missing, f"declared in include/*.h but not exported: {missing}"


def test_library_exports_reference_named_entry_points():
    # kernels::stokeslet_direct_gpu_impl / stresslet_direct_gpu_impl, include/kernels.hpp:17-20 of the reference
    L = C.CDLL(skb.library_path())
    for sym in ("_ZN7kernels25stokeslet_direct_gpu_implEPKdS1_iS1_Pdi",
                "_ZN7kernels25stresslet_direct_gpu_implEPKdS1_iS1_Pdi"):
        assert hasattr(L, sym), sym


def test_python_binding_covers_header():
    skb.library()
    missing = [n for n in _declared_functions() if n not in capi.BOUND_FUNCTIONS]
    assert not missing, f"declared in include/*.h but without a ctypes signature in capi.py: {missing}"


def test_no_cpu_fallback_without_gpu():
    if capi.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(skb.SkbError, match="no CPU fallback"):
        skb.Context(1)
    with pytest.raises(skb.SkbError):
        skb.stokeslet_direct(np.zeros((2, 3)), np.zeros((2, 3)), np.zeros((2, 3)))


def test_product_never_imports_oracle():
    # the oracle is test infrastructure: nothing under skellysim_b200/ or include/ may reference it
    bad = []
    for base in ("skellysim_b200", "include"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".cpp", ".hpp", ".h", "Makefile")):
                    txt = open(os.path.join(dirpath, f), errors="ignore").read()
                    if re.search(r"\boracle\b", txt):
                        bad.append(os.path.join(dirpath, f))
    assert not bad, bad


def test_device_resources_are_released_only_by_their_owners():
    # every stream, event, graph exec, device or pinned allocation and IPC mapping of the library is held by an owner
    # type of skb_internal.hpp (DevBuf, Owned) that releases it; a release call anywhere else is a hand-written teardown
    # list that can fall out of step with the structs.  (The process-lifetime objects -- the pinned upload ring, the
    # default context, prepare_device's table -- are never released: static destructors would run after the CUDA
    # runtime's own teardown at exit.)
    release = re.compile(r"\b(cudaFree|cudaFreeHost|cudaEventDestroy|cudaStreamDestroy|cudaGraphExecDestroy|"
                         r"cudaIpcCloseMemHandle)\b")
    bad = []
    for base in ("skellysim_b200", "include"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if f == "skb_internal.hpp" or not f.endswith((".cu", ".cuh", ".cpp", ".hpp", ".h")):
                    continue
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                txt = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group().count("\n"), txt, flags=re.S)
                for i, line in enumerate(txt.splitlines(), 1):
                    if release.search(line.split("//")[0]):
                        bad.append(f"{f}:{i}: {line.strip()}")
    assert not bad, bad


def test_null_handles_are_refused_before_any_cuda_call():
    # argument errors come back as codes with a message (never a crash), GPU or not
    L = capi.library()
    null = C.c_void_p()
    calls = [
        lambda: L.skb_flow_set_fiber_class(null, 8, None, None),
        lambda: L.skb_flow_set_fiber_operators(null, None, None, None, None, None),
        lambda: L.skb_flow_set_fiber_preconditioner(null, None),
        lambda: L.skb_flow_apply_fiber_force(null, None, None),
        lambda: L.skb_flow_fiber_matvec(null, None, None, None, None),
        lambda: L.skb_flow_apply_fiber_preconditioner(null, None, None),
        lambda: L.skb_flow_apply_matvec(null, None, None, None, None, None, 1.0, None, None, None),
        lambda: L.skb_flow_apply_matvec_dense(null, null, None, None, None, None, None, 1.0, None, None, None),
        lambda: L.skb_flow_set_target_ranges(null, 0, 0, 0, 0, 0, 0),
        lambda: L.skb_flow_apply_fiber_force_device(null, None, None, None),
        lambda: L.skb_flow_fiber_matvec_device(null, None, None, None, None, None),
        lambda: L.skb_dense_apply_device(null, 0, None, None, None, None),
    ]
    for call in calls:
        assert call() != 0
        assert len(L.skb_last_error_string()) > 0


def test_flow_piece_bookkeeping_of_the_binding():
    # capi.Flow._pieces mirrors prepare_matvec_targets (skb_matvec.cu): window and range modes
    f = capi.Flow.__new__(capi.Flow)
    f._h = None
    f.n_fib, f.n_shell, f.n_body = 100, 50, 20
    f._fiber_off = np.array([0, 10, 30, 60, 100])
    assert f._pieces() == (100, 50, 20)
    f._window, f._ranges = (5, 120), None
    assert f._pieces() == (95, 20, 0)
    f._window = (110, -1)
    assert f._pieces() == (0, 40, 20)
    f._ranges, f._window = (1, 3, 10, 20, 0, 20), None
    assert f._pieces() == (50, 10, 20)
    f._ranges = (2, 9, 40, 90, 5, 5)
    assert f._pieces() == (70, 10, 0)

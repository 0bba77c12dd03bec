"""CPU tests of the device build of the per-fiber operators (skb_flow_build_fiber_operators and friends,
include/skelly_b200_flow.h): every new entry point refuses a NULL handle with a message, and the binding's
skb_fiber_params record has the header's layout."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from skellysim_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_new_entry_points_refuse_null_handles():
    L = capi.library()
    null = C.c_void_p()
    D = np.zeros(64)
    p = capi.fiber_params(1, 1.0, 1.0, 0.01, 500.0, 1.0, 0, 0)
    calls = [
        lambda: L.skb_flow_set_fiber_class_derivatives(null, 8, capi._p(D), capi._p(D), capi._p(D)),
        lambda: L.skb_flow_build_fiber_operators(null, capi._params_ptr(p), 1e-2, 1.0),
        lambda: L.skb_flow_get_fiber_operators(null, None, None, None, None),
        lambda: L.skb_mflow_set_fiber_class_derivatives(null, 8, capi._p(D), capi._p(D), capi._p(D)),
        lambda: L.skb_mflow_build_fiber_operators(null, capi._params_ptr(p), 1e-2, 1.0),
    ]
    for call in calls:
        assert call() != 0
        assert b"NULL" in L.skb_last_error_string()


def test_fiber_params_layout_matches_header(tmp_path):
    assert C.sizeof(capi.FiberParams) == 48
    assert capi.FIBER_PARAMS_DTYPE.itemsize == 48
    offsets = {name: getattr(capi.FiberParams, name).offset for name, _ in capi.FiberParams._fields_}
    assert offsets == {name: capi.FIBER_PARAMS_DTYPE.fields[name][1] for name in capi.FIBER_PARAMS_DTYPE.names}
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler to read the header's layout")
    src = tmp_path / "layout.c"
    fields = [name for name, _ in capi.FiberParams._fields_]
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "skelly_b200_flow.h"\nint main(void) {\n'
                   '  printf("%zu\\n", sizeof(skb_fiber_params));\n'
                   + "".join(f'  printf("%zu\\n", offsetof(skb_fiber_params, {f}));\n' for f in fields)
                   + "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [48] + [offsets[f] for f in fields]


def test_fiber_params_from_scalars_and_arrays():
    p = capi.fiber_params(3, [1.0, 2.0, 3.0], 2.5e-3, 0.0125, 500.0, 1.0, [1, 0, 1], 0)
    assert p["length_prev"].tolist() == [1.0, 2.0, 3.0]
    assert p["radius"].tolist() == [0.0125] * 3
    assert p["minus_clamped"].tolist() == [1, 0, 1] and p["plus_hinged"].tolist() == [0, 0, 0]
    with pytest.raises(ValueError, match="length_prev"):
        capi.fiber_params(3, [1.0, 2.0], 1.0, 1.0, 1.0, 1.0, 0, 0)

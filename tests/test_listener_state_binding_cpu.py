"""CPU tests of the ctypes binding of skb_flow_set_listener_state(_device) (capi.set_listener_state,
capi.set_listener_state_device, timestep.Stepper.set_listener_state), with the recorder of test_capi_binding_cpu.py in
place of the library: every call is checked against its declared C signature and recorded by value.  Only a capi.Flow
reaches the C calls; a MultiFlow is refused before any library call, and a Stepper offers only an installed step."""
import numpy as np
import pytest

from skellysim_b200 import capi, timestep
from test_capi_binding_cpu import DT, ETA, _drive, _inputs, _twin_calls, calls  # noqa: F401 (the fixture)


def _set_up(obj, calls, s):
    _drive(obj, calls, [c for c in _twin_calls(s) if c[0] not in ("step", "stats")])


def test_the_state_calls_are_marshalled_as_declared(calls):
    s = _inputs(5)
    fl = capi.Flow(0)
    _set_up(fl, calls, s)
    p = s["params"]
    tension = np.arange(fl.n_fib, dtype=np.float64)
    x = s["x"]
    assert x.shape == (fl.solution_size(),)
    radii = np.array([[0.4, 0.4, 0.4], [0.5, 0.6, 0.7]])
    n0 = len(calls)
    capi.set_listener_state(fl, *p, DT, ETA, tension, x, [1, 2], radii, periphery_interaction=True)
    (name, args), = calls[n0:]
    assert name == "skb_flow_set_listener_state"
    params = capi.fiber_params(2, *p)
    assert args[1] == (params.dtype.str, params.tobytes())
    assert args[2:4] == (DT, ETA)
    assert args[4] == ("<f8", tension.tobytes()) and args[5] == ("<f8", x.tobytes())
    assert args[6] == ("<i4", np.array([1, 2], dtype=np.int32).tobytes())
    assert args[7] == ("<f8", radii.tobytes()) and args[8] == 1
    n0 = len(calls)
    capi.set_listener_state_device(fl, *p, DT, ETA, 0x100, 0x200, [0, 1], radii, stream=0x300)
    (name, args), = calls[n0:]
    assert name == "skb_flow_set_listener_state_device"
    assert args[4:6] == (0x100, 0x200) and args[8] == 0 and args[9] == 0x300
    # the host form checks the sizes it sends; neither form sends a wrong body count
    for bad in (dict(tension=tension[:-1]), dict(x=x[:-1])):
        kw = dict(tension=tension, x=x)
        kw.update(bad)
        with pytest.raises(ValueError):
            capi.set_listener_state(fl, *p, DT, ETA, kw["tension"], kw["x"], [1, 2], radii)
    with pytest.raises(ValueError):
        capi.set_listener_state_device(fl, *p, DT, ETA, 0x100, 0x200, [1], radii[:1])
    assert len(calls) == n0 + 1
    fl.close()


def test_a_multiflow_is_refused_before_any_call(calls):
    s = _inputs(6)
    mf = capi.MultiFlow(2)
    _set_up(mf, calls, s)
    p = s["params"]
    n0 = len(calls)
    with pytest.raises(TypeError, match="capi.Flow"):
        capi.set_listener_state(mf, *p, DT, ETA, np.zeros(mf.n_fib), s["x"], [1, 2], np.ones((2, 3)))
    with pytest.raises(TypeError, match="capi.Flow"):
        capi.set_listener_state_device(mf, *p, DT, ETA, 0x100, 0x200, [1, 2], np.ones((2, 3)))
    st = timestep.Stepper(mf, None, p, ETA)
    st.step(DT)
    n0 = len(calls)
    with pytest.raises(TypeError, match="capi.Flow"):
        st.set_listener_state([1, 2], np.ones((2, 3)))
    assert len(calls) == n0
    mf.close()


def test_a_stepper_offers_only_an_installed_step(calls):
    s = _inputs(7)
    fl = capi.Flow(0)
    _set_up(fl, calls, s)
    st = timestep.Stepper(fl, None, s["params"], ETA)
    with pytest.raises(RuntimeError, match="no installed step"):
        st.set_listener_state([1, 2], np.ones((2, 3)))
    st.backup()
    st.step(DT)  # (the recorder leaves the step's info zero: a finite fiber_error, installed)
    n0 = len(calls)
    st.set_listener_state([1, 2], np.ones((2, 3)))
    assert [c[0] for c in calls[n0:]] == ["skb_flow_set_listener_state"]
    st.restore()  # the restored geometry is not that step's
    with pytest.raises(RuntimeError, match="no installed step"):
        st.set_listener_state([1, 2], np.ones((2, 3)))
    # a step that was not installed (NaN fiber_error) is not kept either
    fl.step = lambda *a, **k: (s["x"], np.zeros(fl.n_fib), dict(fiber_error=np.nan, converged=0))
    st.step(DT)
    with pytest.raises(RuntimeError, match="no installed step"):
        st.set_listener_state([1, 2], np.ones((2, 3)))
    del fl.step
    fl.close()

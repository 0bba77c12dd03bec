"""CPU tests of the ctypes binding's marshalling (no GPU): the library is replaced by a recorder that checks each call's
arguments against the declared C signature, records them by value (arrays by their bytes) and returns 0.  Every public
method of Flow and MultiFlow is driven; the calls a Flow and a MultiFlow make for the same inputs must agree, and so
must a Flow's group_ set-up calls and their plain twins."""
import ctypes as C

import numpy as np
import pytest

from skellysim_b200 import capi

ETA, DT = 0.9, 0.01
FIBER_N, BODY_N = [6, 8], [3, 4]


class _Recorder:
    """the library's stand-in: checks every call against the real library's argtypes, records (symbol, values) and
    returns 0; a create call gets a distinct non-NULL handle"""

    def __init__(self, real):
        self.real, self.calls, self.handles = real, [], []

    def __getattr__(self, name):
        argtypes = getattr(self.real, name).argtypes

        def call(*args):
            assert len(args) == len(argtypes), f"{name}: {len(args)} arguments, declared {len(argtypes)}"
            for a, t in zip(args, argtypes):
                t.from_param(a)  # raises as the real call would on an argument of the wrong kind
            if name.endswith(("_create", "_create_on")):
                self.handles.append(args[-1]._obj)
                self.handles[-1].value = 0x1000 * len(self.handles)
            self.calls.append((name, tuple(_value(a) for a in args)))
            return 0
        return call


def _value(a):
    if a is None or isinstance(a, (int, float, bytes)):
        return a
    if hasattr(a, "_arr"):  # a pointer numpy made with .ctypes.data_as: the array's bytes
        return a._arr.dtype.str, a._arr.tobytes(order="A")
    if isinstance(a, type(C.byref(C.c_int()))):
        a = a._obj
    if isinstance(a, C.Structure):
        return tuple(_value(getattr(a, f)) for f, _ in a._fields_)
    if isinstance(a, C.Array):
        return tuple(a)
    if isinstance(a, C.c_void_p) and a._objects:  # a host buffer cast to void *: its bytes
        return tuple(bytes(o) for o in a._objects.values())
    return a.value


class _ZeroedNumpy:
    """numpy with zero-filled empty() / empty_like(): the output buffers the binding allocates record the same bytes
    on every run"""
    empty, empty_like = staticmethod(np.zeros), staticmethod(np.zeros_like)

    def __getattr__(self, name):
        return getattr(np, name)


@pytest.fixture
def calls(monkeypatch):
    rec = _Recorder(capi.library())
    monkeypatch.setattr(capi, "_lib", rec)
    monkeypatch.setattr(capi, "np", _ZeroedNumpy())
    yield rec.calls
    for h in rec.handles:  # no made-up handle may reach the real library's destroy calls
        h.value = None


def _inputs(seed=0):
    rng = np.random.default_rng(seed)
    r = lambda *shape: rng.normal(size=shape)
    nf, nb, n_fib, n_body = len(FIBER_N), len(BODY_N), sum(FIBER_N), sum(BODY_N)
    body_sq = [r(3 * n + 6, 3 * n + 6) for n in BODY_N]
    return dict(
        fibers=(r(n_fib, 3), FIBER_N, [1.0, 1.5]), shell=(r(5, 3), r(5, 3)), bodies=(r(n_body, 3), r(n_body, 3), r(nb, 3)),
        classes=[(n, r(n, n), r(4 * n - 14, 4 * n), r(n, n), r(n, n), r(n, n)) for n in FIBER_N],
        params=(r(nf) ** 2, 2.5e-3, 0.0125, 500.0, 1.0, [0, 1], 0),
        A=[r(4 * n, 4 * n) for n in FIBER_N], force=[r(3 * n, 4 * n) for n in FIBER_N], xs=r(n_fib, 3),
        node_f=r(n_fib, 3), shell_d=r(5, 3), body_d=r(n_body, 3), ft=r(nb, 6), trg=r(4, 3), per_fiber=r(nf),
        body_ops=(BODY_N, r(n_body), r(n_body, 3), r(n_body, 3), r(n_body, 3), body_sq),
        frames=(BODY_N, r(n_body, 3), r(n_body, 3), r(n_body), r(n_body, 3), r(n_body, 3), r(n_body, 3), body_sq),
        place=(r(nb, 3), r(nb, 4)), links=([0, -1], r(nf, 3), 0.01), x=r(4 * n_fib + 15 + sum(3 * n + 6 for n in BODY_N)))


def _twin_calls(s):
    """(method, args, kwargs) of every method Flow and MultiFlow share, in an order that sets up what later calls use"""
    p = s["params"]
    out = [("set_fibers", s["fibers"], {}), ("set_periphery", s["shell"], {}), ("set_bodies", s["bodies"], {}),
           ("set_self_exclusion", (True,), {}), ("set_cross", (1,), {}), ("set_overlap", (False,), {})]
    for n, D1, P, D2, D3, D4 in s["classes"]:
        out += [("set_fiber_class", (n, D1, P), {}), ("set_fiber_class_derivatives", (n, D2, D3, D4), {})]
    rhs_kw = dict(v_growth=s["per_fiber"], force_scale=0.5)
    out += [
        ("set_fiber_preconditioner", (s["A"],), {}),
        ("build_fiber_operators", (*p, DT, ETA), {}),
        ("build_fiber_rhs", (*p, DT, ETA), dict(rhs_kw, v_on_fibers=s["node_f"], f_external=s["node_f"])),
        ("build_fiber_rhs", (*p, DT, ETA), {}),
        ("matvec", (s["node_f"], s["shell_d"], s["body_d"], s["ft"], ETA), {}),
        ("set_point_sources", (s["trg"][:2], s["trg"][1:3], s["trg"][2:]), {}),
        ("set_background", ([0, 1, 2], [1.0, 2.0, 3.0], [0.1, 0.2, 0.3]), {}),
        ("velocity_at_targets", (s["trg"], s["node_f"], s["shell_d"], s["body_d"], s["ft"], ETA), {}),
        ("set_body_operators", s["body_ops"], {}),
        ("set_body_operators", s["body_ops"][:5], {}),
        ("set_body_frames", s["frames"], {}),
        ("place_bodies", s["place"], {}),
        ("set_fiber_links", s["links"], {}),
        ("set_fiber_links", (), {}),
        ("set_periphery_shape", (capi.PERIPHERY_ELLIPSOID, 5.0, 4.0, 3.0), dict(fiber_minus_clamped=[0, 1],
                                                                                 body_radius=[0.5, 0.0])),
        ("set_periphery_shape", (capi.PERIPHERY_SPHERE, 5.0), dict(binding_active=True)),
        ("build_system_rhs", (*p, DT, ETA), dict(rhs_kw, f_external=s["node_f"], body_forces_torques=s["ft"])),
        ("set_gmres", (50,), {}),
        ("solution_size", (), {}),
        ("step", (*p, DT, ETA), dict(rhs_kw, f_external=s["node_f"], body_forces_torques=s["ft"], fiber_body=[0, -1],
                                     site_ref=s["links"][1], tol=1e-8, num_blocks=20, max_iters=30)),
        ("step", (*p, DT, ETA), {}),
        ("fibers", (), {}), ("placement", (), {}), ("stats", (), {}),
    ]
    return out


def _drive(obj, calls, table):
    """runs the table on obj; returns per entry the library calls it made"""
    per = []
    for name, args, kw in table:
        n0 = len(calls)
        getattr(obj, name)(*args, **kw)
        per.append(calls[n0:])
    return per


def _public(cls):
    return {n for n in dir(cls) if not n.startswith("_") and callable(getattr(cls, n))}


def test_flow_and_multiflow_make_the_same_calls(calls):
    s = _inputs()
    table = _twin_calls(s)
    fl, mf, dense = capi.Flow(0), capi.MultiFlow([0, 1]), capi.Dense(1)
    got_f = _drive(fl, calls, table)
    got_m = _drive(mf, calls, table)
    fl.step(*s["params"], DT, ETA, dense=dense)
    step_dense = calls[-1]
    assert len(table) > 30 and any(got_f)
    for (name, _, _), cf, cm in zip(table, got_f, got_m):
        assert len(cf) == len(cm), name
        for (sf, af), (sm, am) in zip(cf, cm):
            assert sf.startswith("skb_flow_") and sm == "skb_mflow_" + sf[len("skb_flow_"):], (name, sf, sm)
            assert af[0] == fl._h.value and am[0] == mf._h.value, name
            if name == "step":  # skb_flow_step alone takes the Dense handle after the flow's
                assert af[1] is None
                af = af[:1] + af[2:]
            assert af[1:] == am[1:], name
    assert step_dense[0] == "skb_flow_step" and step_dense[1][1] == dense._h.value
    # the readbacks and the bookkeeping agree as well
    assert fl.solution_size() == mf.solution_size() and mf.n_fibers == fl._n_fibers() == len(FIBER_N)
    assert mf._pieces() == fl._pieces() and mf._own_fibers() == fl._own_fibers()


@pytest.mark.parametrize("group, plain", [
    ("group_set_body_operators", "set_body_operators"), ("group_set_body_frames", "set_body_frames"),
    ("group_place_bodies", "place_bodies"), ("group_set_fiber_links", "set_fiber_links")])
def test_group_setup_calls_marshal_as_their_plain_twins(calls, group, plain):
    s = _inputs(1)
    args = dict(set_body_operators=s["body_ops"], set_body_frames=s["frames"], place_bodies=s["place"],
                set_fiber_links=s["links"])[plain]
    fl = capi.Flow(0)
    fl.set_bodies(*s["bodies"])
    n0 = len(calls)
    getattr(fl, plain)(*args)
    sol = fl.solution_size()
    getattr(fl, group)(*args)
    (sp, ap), (sg, ag) = calls[n0:]
    assert sp == "skb_flow_" + plain and sg == "skb_flow_" + group and ap == ag
    assert fl.solution_size() == sol


def test_a_flows_calls_cover_its_own_fibers(calls):
    # with target ranges, the per-fiber tables and the fiber rows are those of the own fibers
    s = _inputs(2)
    fl = capi.Flow(0)
    fl.set_fibers(*s["fibers"])
    fl.set_target_ranges(1, 2, 0, 0, 0, 0)
    own = (1.5, 2.5e-3, 0.0125, 500.0, 1.0, [1], 0)  # the second fiber's parameters
    fl.build_fiber_operators(*own, DT, ETA)
    assert len(calls[-1][1][1][1]) == capi.FIBER_PARAMS_DTYPE.itemsize  # one fiber's skb_fiber_params
    with pytest.raises(ValueError):
        fl.build_fiber_operators(*s["params"], DT, ETA)
    rhs = fl.build_fiber_rhs(*own, DT, ETA)
    assert rhs.shape == (4 * FIBER_N[1],)
    assert fl.matvec(s["node_f"], np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 6)), ETA).shape == (FIBER_N[1], 3)


def test_every_method_of_the_binding_is_marshalled_as_declared(calls):
    s = _inputs(3)
    p = s["params"]
    table = _twin_calls(s)
    dense = capi.Dense(1)
    d = [0x10 * (k + 1) for k in range(12)]  # device addresses
    own = (1.0,) + p[1:5] + (1, 0)  # one fiber's parameters, once target ranges own the first fiber
    flow_only = [
        ("fiber_flow", (s["trg"], s["node_f"], ETA), {}), ("periphery_flow", (s["trg"], s["shell_d"], ETA), {}),
        ("body_flow", (s["trg"], s["body_d"], s["ft"], ETA), {}),
        ("set_listener_frame", (s["node_f"], s["shell_d"], s["body_d"], s["ft"], s["ft"], [1, 2], s["place"][0], ETA),
         {}),
        ("velocity_field", (s["trg"],), {}),
        ("streamlines", (s["trg"],), dict(max_points=5)), ("vortexlines", (s["trg"][:2],), dict(back_integrate=False)),
        ("matvec_device", (*d[:5], ETA, d[5]), dict(stream=d[6])),
        ("set_fiber_operators", (s["A"], s["force"], s["xs"], [1.0, 1.5], [0, 1]), {}),
        ("set_fiber_operators", (np.concatenate([a.ravel(order="F") for a in s["A"]]),
                                 np.concatenate([f.ravel(order="F") for f in s["force"]]), s["xs"], [1.0, 1.5],
                                 [0, 1]), dict(colmajor=True)),
        ("build_fiber_rhs_device", (*p, DT, ETA, d[0], 0, d[2]), dict(v_growth=0.1, stream=d[3])),
        ("get_fiber_operators", (), {}), ("get_fiber_operators", (), dict(inverse=False)),
        ("apply_fiber_preconditioner", (s["x"][:4 * 14],), {}),
        ("apply_fiber_preconditioner_device", (d[0], d[1]), dict(stream=d[2])),
        ("apply_fiber_force", (s["x"][:4 * 14],), {}), ("apply_fiber_force_device", (d[0], d[1]), {}),
        ("fiber_matvec", (s["x"][:4 * 14], s["node_f"]), dict(v_fib_boundary=s["x"][:14].reshape(2, 7))),
        ("fiber_matvec_device", (d[0], d[1], 0, d[3]), {}),
        ("apply_matvec", (s["x"][:4 * 14], s["shell_d"], s["body_d"], s["ft"], ETA), dict(dense=dense)),
        ("apply_matvec", (s["x"][:4 * 14], s["shell_d"], s["body_d"], s["ft"], ETA),
         dict(fiber_link_conditions=s["x"][:14].reshape(2, 7))),
        ("apply_matvec_device", (dense, *d[:6], ETA, *d[6:9]), dict(stream=d[9])),
        ("apply_matvec_device", (None, d[0], 0, 0, 0, 0, 0, ETA, d[6], 0, 0), {}),
        ("get_body_operators", (), {}),
        ("apply_system_matvec", (s["x"], ETA), dict(dense=dense)),
        ("apply_system_matvec_device", (dense, d[0], ETA, d[1]), dict(stream=d[2])),
        ("apply_system_preconditioner", (s["x"],), {}),
        ("apply_system_preconditioner_device", (None, d[0], d[1]), {}),
        ("build_system_rhs_device", (*p, DT, ETA, d[0], d[1], 0, d[3]), dict(force_scale=s["per_fiber"])),
        ("solve_system", (s["x"], ETA), dict(dense=dense, tol=1e-9, num_blocks=10, max_iters=7)),
        ("solve_system_device", (dense, d[0], ETA, d[1]), dict(max_iters=3, stream=d[2])),
        ("periphery_interaction", (), {}), ("periphery_interaction", (), dict(n_own_nodes=8, n_own_fibers=1)),
        ("set_nucleation_sites", ([2, 1], s["trg"][:3]), {}),
        ("step_flags", (), {}), ("fiber_error", (), {}), ("last_sym_kernel", (), {}),
        ("set_target_window", (3, 20), {}), ("set_target_ranges", (0, 1, 0, 5, 2, 7), {}),
        ("group_init", (0, 2), {}), ("group_export", (), {}), ("group_import", (1, bytes(range(64))), {}),
        ("group_connect", (1, capi.Flow(0)), {}), ("group_warmup", (), {}), ("group_set_solo", (True,), {}),
        ("group_error", (), {}),
        ("group_set_body_operators", s["body_ops"], {}), ("group_set_body_frames", s["frames"], {}),
        ("group_place_bodies", s["place"], {}), ("group_set_fiber_links", ([1], s["trg"][:1], [0.02]), {}),
        ("group_apply_system_matvec_device", (dense, d[0], ETA, d[1]), dict(stream=d[2])),
        ("group_apply_system_preconditioner_device", (None, d[0], d[1]), {}),
        ("group_solve_system_device", (dense, None, d[0], ETA, d[1]), dict(num_blocks=4, max_iters=5)),
        ("group_build_system_rhs_device", (*own, DT, ETA, d[0], 0, 0, d[3]), {}),
        ("group_step_device", (*own, DT, ETA),
         dict(dense_matvec=dense, d_f_external=d[0], fiber_body=[0], site_ref=s["trg"][:1], d_x_local=d[1])),
        ("dynamic_instability", ({"n_nodes": 8, "v_growth": 0.1, "nucleation_rate": 2.0}, DT, 7, 3, p,
                                 [[0, 1], [-1, -1]], [0, 1]), {}),
        ("close", (), {}), ("close", (), {}),
    ]
    mflow_only = [
        ("partition", (1,), {}), ("set_fiber_operators", (s["A"], s["force"], s["xs"], [1.0, 1.5], [0, 1]), {}),
        ("set_dense", (capi.DENSE_M_INV, s["x"][:25].reshape(5, 5)), {}),
        ("apply_matvec", (s["x"][:4 * 14], s["shell_d"], s["body_d"], s["ft"], ETA), {}),
        ("periphery_interaction", (), {}),
        ("apply_system_matvec", (s["x"], ETA), {}), ("apply_system_preconditioner", (s["x"],), {}),
        ("solve_system", (s["x"], ETA), dict(num_blocks=5)),
        ("close", (), {}), ("close", (), {}),
    ]
    for cls, table_own in ((capi.Flow, flow_only), (capi.MultiFlow, mflow_only)):
        obj = cls(0) if cls is capi.Flow else cls(2)
        full = table + table_own
        assert {name for name, _, _ in full} == _public(cls), "every public method is driven"
        per = _drive(obj, calls, full)
        assert obj._h.value is None
        destroys = [c for c in calls if c[0] == f"skb_{'flow' if cls is capi.Flow else 'mflow'}_destroy"]
        assert len(destroys) == 1  # closing twice releases once
        for (name, _, _), made in zip(full, per):
            assert made or name in ("solution_size", "close", "_n_fibers"), f"{name} made no call"

"""Time stepping of a whole system: System::step (system.cpp:482-492) through capi.Flow.step, and the acceptance logic
of System::run (system.cpp:515-568) around it.

The fiber-periphery repulsion, the periphery binding and the collision test run inside the step once the flow has a
periphery shape (Flow.set_periphery_shape): the step reports the collision test as info["collided"].  The bodies' force
schedule stays the caller's host code (DESIGN.md §7): `run` takes it as the callable `forces(time, r_fib)`, and a
caller's own `collided(r_fib, centers)` still replaces the step's test.

With dynamic_instability (the [dynamic_instability] table as a dict), each step of `run` starts as
System::prep_state_for_solver does: Stepper.dynamic_instability removes, grows and nucleates fibers on the device
(Flow.dynamic_instability) before the forces are asked for, and the Stepper carries its per-fiber tables to the new fiber
set.  Its random stream is (seed, call counter): the counter advances on every attempt and a rejected step does not
rewind it, as the reference's restore() does not rewind its generator.

A run on the device can be observed on the device: `run` calls `observe(time, stepper, info)` after every accepted step,
and Stepper.set_listener_state sets the flow's listener frame from the step it kept (the installed geometry, the step's
solution and tension), so that the flow's velocity_field, streamlines and vortexlines answer on the state the step
just installed, as the reference's listener does on a trajectory frame.

One deviation from the reference's loop (DESIGN.md §5): the reference sets dt to the grown dt_new before it advances
time on an accepted step (system.cpp:554-557), so time advances by a dt no step used.  Here time advances by the dt of
the step that was accepted."""
import numpy as np

from . import capi

class Stepper:
    """A capi.Flow or capi.MultiFlow and what its steps need: its Dense (None without periphery), the fibers' parameters (the seven of
    Flow.build_fiber_operators, scalars or per fiber), eta, the fibers' bindings (fiber_body, -1 free, and site_ref, the
    body-frame nucleation sites) and the solve's settings.  The flow holds the geometry; backup / restore keep a host
    copy of it: fiber positions, body centres and quaternions."""

    def __init__(self, flow, dense, params, eta, fiber_body=None, site_ref=None, v_growth=None, force_scale=None,
                 tol=1e-10, num_blocks=300, max_iters=1000, dynamic_instability=None, seed=0, fiber_site=None):
        """dynamic_instability: None (off) or a dict of the [dynamic_instability] table (capi.DynamicInstability's
        fields); then the flow needs Flow.set_nucleation_sites, each bound fiber names its site by fiber_site (the
        index among its body's sites) instead of site_ref, and seed starts the random stream."""
        self.flow, self.dense, self.params, self.eta = flow, dense, tuple(params), float(eta)
        self.fiber_body, self.site_ref = fiber_body, site_ref
        self.v_growth, self.force_scale = v_growth, force_scale
        self.tol, self.num_blocks, self.max_iters = tol, num_blocks, max_iters
        self._backup = None
        self.last = None  # (x, tension, dt) of the installed step: its solution vector, fiber tensions and timestep
        self.di, self.seed, self.counter = dynamic_instability, int(seed), 0
        if self.di is not None:
            n = flow._n_fibers()
            p = capi.fiber_params(n, *self.params)
            self.params = tuple(p[name].copy() for name in capi.FIBER_PARAMS_DTYPE.names)
            body = np.full(n, -1, dtype=np.int32) if fiber_body is None else np.asarray(fiber_body, dtype=np.int32)
            site = np.full(n, -1, dtype=np.int32) if fiber_site is None else np.asarray(fiber_site, dtype=np.int32)
            self.binding = np.stack([body, np.where(body >= 0, site, -1)], axis=1).astype(np.int32)
            self.v_growth = np.zeros(n) if v_growth is None else capi._per_fiber(v_growth, n)
            self.force_scale = None if force_scale is None else capi._per_fiber(force_scale, n)
            self.plus_pinned = np.asarray(p["plus_hinged"], dtype=np.int32).copy()
            self._bindings()

    def positions(self):
        return self.flow.fibers()

    def placement(self):
        if self.flow.n_bodies == 0:
            return np.zeros((0, 3)), np.zeros((0, 4))
        return self.flow.placement()

    def _bindings(self):
        """fiber_body and site_ref of the step from the (body, site) bindings and the flow's site table"""
        body = self.binding[:, 0]
        self.fiber_body = body.copy()
        if not (body >= 0).any():
            self.site_ref = None
            return
        counts, ref = self.flow._sites
        off = np.concatenate([[0], np.cumsum(counts)])
        flat = np.where(body >= 0, off[np.maximum(body, 0)] + self.binding[:, 1], 0)
        self.site_ref = ref[flat]

    def dynamic_instability(self, dt):
        """System::dynamic_instability before a step (a no-op without the model); returns the call's dict or None"""
        if self.di is None:
            return None
        call = self.counter
        self.counter += 1
        out = self.flow.dynamic_instability(self.di, dt, self.seed, call, self.params, self.binding, self.plus_pinned)
        if out["v_growth"] is None:  # n_nodes == 0: nothing changed
            return out
        o = out["origin"]
        carry = lambda a: np.where(o >= 0, a[np.maximum(o, 0)] if a.size else 0, 0).astype(a.dtype)
        self.params = tuple(out["params"][name].copy() for name in capi.FIBER_PARAMS_DTYPE.names)
        self.binding = out["binding"].astype(np.int32)
        self.v_growth = out["v_growth"]
        if self.force_scale is not None:
            self.force_scale = carry(self.force_scale)
        self.plus_pinned = carry(self.plus_pinned)
        self._bindings()
        return out

    def step(self, dt, f_external=None, body_forces_torques=None):
        """one System::step; returns the step's info (the solve's fields, fiber_error, worst_fiber; a NaN fiber_error:
        the solution was not finite and nothing was installed)"""
        x, tension, info = self.flow.step(*self.params, dt, self.eta, dense=self.dense, f_external=f_external,
                                    body_forces_torques=body_forces_torques, fiber_body=self.fiber_body,
                                    site_ref=self.site_ref, v_growth=self.v_growth, force_scale=self.force_scale,
                                    tol=self.tol, num_blocks=self.num_blocks, max_iters=self.max_iters)
        # kept only for a step whose geometry is installed: the frame pairs that geometry with this solution
        self.last = (x, tension, float(dt)) if np.isfinite(info["fiber_error"]) else None
        if self.di is not None and np.isfinite(info["fiber_error"]):
            self.plus_pinned = self.flow.step_flags()
        return info

    def set_listener_state(self, body_kind=None, body_radii=None, periphery_interaction=False):
        """The flow's listener frame from the last step (capi.set_listener_state): the installed geometry, the
        step's solution and tension, the fiber parameters and dt it was taken with.  body_kind / body_radii as
        Flow.set_listener_frame (None without bodies).  A capi.Flow only (the listener is single-device).  Refused
        without an installed step: before the first step, after a step that was not installed, after restore()."""
        if not isinstance(self.flow, capi.Flow):
            raise TypeError(f"set_listener_state: the listener's frame needs a capi.Flow (one device), not a "
                            f"{type(self.flow).__name__}")
        if self.last is None:
            raise RuntimeError("set_listener_state: no installed step (none was taken, the last one was not "
                               "installed, or it was restored)")
        x, tension, dt = self.last
        capi.set_listener_state(self.flow, *self.params, dt, self.eta, tension, x, body_kind, body_radii,
                                periphery_interaction)

    def backup(self):
        self._backup = (self.positions(), *self.placement())
        if self.di is not None:  # the whole fiber set: counts, lengths, the per-fiber tables, the flags
            shape = getattr(self.flow, "_shape", None)
            self._fiber_set = (np.diff(self.flow._fiber_off), self.flow._lengths.copy(), self.params, self.binding,
                               self.v_growth, self.force_scale, self.plus_pinned,
                               None if shape is None else shape["fiber_minus_clamped"].copy())

    def restore(self):
        r, c, q = self._backup
        self.last = None  # the restored geometry is not the last step's
        if self.di is None:
            self.flow.set_fibers(r, np.diff(self.flow._fiber_off), self.flow._lengths)
        else:
            (n_nodes, lengths, self.params, self.binding, self.v_growth, self.force_scale, self.plus_pinned,
             clamped) = self._fiber_set
            self.flow.set_fibers(r, n_nodes, lengths)
            self._bindings()
            if clamped is not None:
                self.flow.set_periphery_shape(**dict(self.flow._shape, fiber_minus_clamped=clamped))
            self.flow.set_gmres(self.flow._gmres_blocks)
        if self.flow.n_bodies:
            self.flow.place_bodies(c, q)


def run(stepper, t_final, dt, adaptive=True, dt_min=1e-5, dt_max=np.inf, beta_up=1.2, beta_down=0.5,
        fiber_error_tol=0.1, forces=None, collided=None, time=0.0, observe=None):
    """System::run's loop until time >= t_final.  Each step: backup, the dynamic instability (Stepper's model, if
    any), forces(time, r_fib) -> (f_external (N_f, 3),
    F_T (n_bodies, 6)), either None (no callable: no external forces), the step, then the acceptance:
      adaptive: accept when converged and fiber_error <= fiber_error_tol, and then grow dt by beta_up (at most dt_max)
      when fiber_error <= 0.9 fiber_error_tol; otherwise shrink dt by beta_down.  A converged step that collided is
      rejected with dt halved (system.cpp:542-546): collided(r_fib, centers) decides when given, else the step's
      info["collided"].  A dt below dt_min raises RuntimeError.
      not adaptive: every step is accepted, dt stays; a step that was not installed (NaN fiber_error) raises.
    A rejected step is restored.  observe(time, stepper, info), when given, is called after every accepted step with the
    advanced time, while that step's geometry is installed (Stepper.set_listener_state then sets the listener's frame of
    it); it changes nothing of the loop.  Returns (time, dt, log): log one (time, dt used, accepted, fiber_error) per step."""
    log = []
    while time < t_final:
        stepper.backup()
        if hasattr(stepper, "dynamic_instability"):  # (distributed.RankStepper and other steppers have no model)
            stepper.dynamic_instability(dt)
        f_ext, ft = forces(time, stepper.positions()) if forces is not None else (None, None)
        info = stepper.step(dt, f_external=f_ext, body_forces_torques=ft)
        converged, err = bool(info["converged"]), info["fiber_error"]
        dt_new, accept = dt, True
        if adaptive:
            accept = converged and err <= fiber_error_tol
            if accept:
                if err <= 0.9 * fiber_error_tol:
                    dt_new = min(dt_max, dt * beta_up)
            else:
                dt_new = dt * beta_down
            if converged and (collided(stepper.positions(), stepper.placement()[0]) if collided is not None
                              else info.get("collided", False)):
                dt_new, accept = dt * 0.5, False
            if dt_new < dt_min:
                raise RuntimeError(f"timestep {dt_new:g} smaller than dt_min = {dt_min:g} at time {time:g} "
                                   f"(fiber_error {err:g})")
        if not adaptive and not np.isfinite(err):
            raise RuntimeError(f"the step at time {time:g} was not finite and was not installed (dt = {dt:g})")
        if accept:
            time += dt
            if observe is not None:
                observe(time, stepper, info)
        else:
            stepper.restore()
        log.append((time, dt, accept, err))
        dt = dt_new
    return time, dt, log

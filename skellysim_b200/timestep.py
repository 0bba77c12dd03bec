"""Time stepping of a whole system: System::step (system.cpp:482-492) through capi.Flow.step, and the acceptance logic
of System::run (system.cpp:515-568) around it.

The fiber-periphery repulsion, the periphery binding and the collision test run inside the step once the flow has a
periphery shape (Flow.set_periphery_shape): the step reports the collision test as info["collided"].  The bodies' force
schedule stays the caller's host code (DESIGN.md §7): `run` takes it as the callable `forces(time, r_fib)`, and a
caller's own `collided(r_fib, centers)` still replaces the step's test.

One deviation from the reference's loop (DESIGN.md §5): the reference sets dt to the grown dt_new before it advances
time on an accepted step (system.cpp:554-557), so time advances by a dt no step used.  Here time advances by the dt of
the step that was accepted."""
import numpy as np

class Stepper:
    """A capi.Flow or capi.MultiFlow and what its steps need: its Dense (None without periphery), the fibers' parameters (the seven of
    Flow.build_fiber_operators, scalars or per fiber), eta, the fibers' bindings (fiber_body, -1 free, and site_ref, the
    body-frame nucleation sites) and the solve's settings.  The flow holds the geometry; backup / restore keep a host
    copy of it: fiber positions, body centres and quaternions."""

    def __init__(self, flow, dense, params, eta, fiber_body=None, site_ref=None, v_growth=None, force_scale=None,
                 tol=1e-10, num_blocks=300, max_iters=1000):
        self.flow, self.dense, self.params, self.eta = flow, dense, tuple(params), float(eta)
        self.fiber_body, self.site_ref = fiber_body, site_ref
        self.v_growth, self.force_scale = v_growth, force_scale
        self.tol, self.num_blocks, self.max_iters = tol, num_blocks, max_iters
        self._backup = None

    def positions(self):
        return self.flow.fibers()

    def placement(self):
        if self.flow.n_bodies == 0:
            return np.zeros((0, 3)), np.zeros((0, 4))
        return self.flow.placement()

    def step(self, dt, f_external=None, body_forces_torques=None):
        """one System::step; returns the step's info (the solve's fields, fiber_error, worst_fiber; a NaN fiber_error:
        the solution was not finite and nothing was installed)"""
        _, _, info = self.flow.step(*self.params, dt, self.eta, dense=self.dense, f_external=f_external,
                                    body_forces_torques=body_forces_torques, fiber_body=self.fiber_body,
                                    site_ref=self.site_ref, v_growth=self.v_growth, force_scale=self.force_scale,
                                    tol=self.tol, num_blocks=self.num_blocks, max_iters=self.max_iters)
        return info

    def backup(self):
        self._backup = (self.positions(), *self.placement())

    def restore(self):
        r, c, q = self._backup
        self.flow.set_fibers(r, np.diff(self.flow._fiber_off), self.flow._lengths)
        if self.flow.n_bodies:
            self.flow.place_bodies(c, q)


def run(stepper, t_final, dt, adaptive=True, dt_min=1e-5, dt_max=np.inf, beta_up=1.2, beta_down=0.5,
        fiber_error_tol=0.1, forces=None, collided=None, time=0.0):
    """System::run's loop until time >= t_final.  Each step: backup, forces(time, r_fib) -> (f_external (N_f, 3),
    F_T (n_bodies, 6)), either None (no callable: no external forces), the step, then the acceptance:
      adaptive: accept when converged and fiber_error <= fiber_error_tol, and then grow dt by beta_up (at most dt_max)
      when fiber_error <= 0.9 fiber_error_tol; otherwise shrink dt by beta_down.  A converged step that collided is
      rejected with dt halved (system.cpp:542-546): collided(r_fib, centers) decides when given, else the step's
      info["collided"].  A dt below dt_min raises RuntimeError.
      not adaptive: every step is accepted, dt stays; a step that was not installed (NaN fiber_error) raises.
    A rejected step is restored.  Returns (time, dt, log): log one (time, dt used, accepted, fiber_error) per step."""
    log = []
    while time < t_final:
        stepper.backup()
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
        else:
            stepper.restore()
        log.append((time, dt, accept, err))
        dt = dt_new
    return time, dt, log

"""Host-side mirror of the reference's Belos adapters for the device-resident path (SURVEY.md 8a row a12).

    reference (src/core/solver_hydro.cpp)                      here
    --------------------------------------------------------  ---------------------------------------------
    A_fiber_hydro::apply   :42-48  -> System::apply_matvec      HydroOperator.apply            (A x)
    P_inv_hydro::apply     :23-40  -> System::apply_preconditioner   HydroOperator.apply_preconditioner (P^-1 x)
    Solver<>::solve        :64-95  (Belos GMRES, caller)        iterate(): the operator sequence of K GMRES
                                                                iterations, nothing else

One GMRES iteration of the reference is `P_inv_hydro::apply` followed by `A_fiber_hydro::apply` (right
preconditioning, solver_hydro.cpp:79-81).  Both are evaluated here with every vector resident on the device: the fiber
block of the preconditioner is a batched GEMV over explicit inverses (skb_flow_apply_fiber_preconditioner_device), the
periphery block a row-block GEMV with M_inv (skb_dense_apply_device), the operator apply is
skb_flow_apply_matvec_device.  HydroOperator leaves the body block to the caller: `apply` hands back the velocities at
the body nodes and takes the body densities / link forces as (small) device tensors.  SystemOperator does not: it
applies A and P^-1 to whole solution vectors [fibers | shell | bodies] with the body block and the fiber-body links on
the device as well (skb_flow_apply_system_matvec_device / _preconditioner_device), and builds the right-hand side of
the solve there too (skb_flow_build_system_rhs_device).

This module sequences calls and owns work vectors; it computes nothing itself.  torch is used for device memory only.
"""
from __future__ import annotations

from . import capi


class HydroOperator:
    """A and P^-1 of the mobility solve for ONE flow (a whole system, or one group member with its own rows).

    flow: capi.Flow with geometry, fiber operators and fiber preconditioner set; dense: capi.Dense on the flow's device
    holding the own rows of stresslet_plus_complementary (and M_inv for the preconditioner) or None; n_* are the OWN
    counts (fiber nodes, periphery rows, body rows)."""

    def __init__(self, flow, dense, n_fib_nodes: int, n_shell_rows: int, n_body_rows: int, eta: float, device,
                 shell_row_begin: int = 0, n_shell_total: int | None = None):
        import torch
        self.torch = torch
        self.flow, self.dense, self.eta = flow, dense, float(eta)
        self.nf, self.ns, self.nb = int(n_fib_nodes), int(n_shell_rows), int(n_body_rows)
        self.s0 = int(shell_row_begin)
        self.ns_total = int(self.ns if n_shell_total is None else n_shell_total)
        kw = dict(dtype=torch.float64, device=device)
        self.res_f = torch.zeros(max(4 * self.nf, 1), **kw)
        self.res_s = torch.zeros((max(self.ns, 1), 3), **kw)
        self.v_b = torch.zeros((max(self.nb, 1), 3), **kw)
        self.y_f = torch.zeros(max(4 * self.nf, 1), **kw)
        self.y_s = torch.zeros((max(self.ns, 1), 3), **kw)
        self.launches = 0

    def _stream(self):
        return self.torch.cuda.current_stream().cuda_stream

    def apply(self, x_f, x_s, body_density, body_forces, body_torques, link=None):
        """A_fiber_hydro::apply (solver_hydro.cpp:42-48) = System::apply_matvec (system.cpp:269-324), fiber and
        periphery rows: returns (res_fibers, res_shell, v_bodies) -- views valid until the next call."""
        p = lambda t: t.data_ptr() if t is not None and t.numel() else 0
        self.flow.apply_matvec_device(self.dense, p(x_f), p(x_s), p(body_density), p(body_forces), p(body_torques),
                                      p(link), self.eta, self.res_f.data_ptr(), self.res_s.data_ptr(),
                                      self.v_b.data_ptr(), self._stream())
        self.launches = self.flow.stats()["launches"]
        return self.res_f[:4 * self.nf], self.res_s[:self.ns], self.v_b[:self.nb]

    def apply_preconditioner(self, x_f, x_s_all):
        """P_inv_hydro::apply (solver_hydro.cpp:23-40) = System::apply_preconditioner (system.cpp:248-262), fiber and
        periphery blocks: y_f = A_^-1 x_f per fiber (fcfd.cpp:331-339), y_s = M_inv x_shell (periphery.cpp:21-30;
        x_s_all is the COMPLETE periphery vector, the result the own rows)."""
        st = self._stream()
        if self.nf:
            self.flow.apply_fiber_preconditioner_device(x_f.data_ptr(), self.y_f.data_ptr(), st)
        if self.ns and self.dense is not None:
            self.dense.apply_device(capi.DENSE_M_INV, x_s_all.data_ptr(), 0, self.y_s.data_ptr(), st)
        return self.y_f[:4 * self.nf], self.y_s[:self.ns]


def iterate(op: HydroOperator, x_f, x_s, body_density, body_forces, body_torques, link, n_iter: int):
    """The operator sequence of `n_iter` right-preconditioned GMRES iterations on a whole system (one flow):
    x <- A P^-1 x, rescaled to unit max-norm on the device so that it neither overflows nor needs a host round trip.
    Returns (x_f, x_s) after the last iteration."""
    torch = op.torch
    for _ in range(n_iter):
        y_f, y_s = op.apply_preconditioner(x_f, x_s)
        r_f, r_s, _ = op.apply(y_f, y_s, body_density, body_forces, body_torques, link)
        scale = torch.maximum(r_f.abs().max() if r_f.numel() else r_s.abs().max(),
                              r_s.abs().max() if r_s.numel() else r_f.abs().max())
        x_f = r_f / scale
        x_s = r_s / scale
    return x_f, x_s


class SystemOperator:
    """A and P^-1 of the whole mobility system on whole solution vectors [fibers | shell | bodies] (get_solution_maps,
    system.cpp:69-92) for ONE single-device flow: A_fiber_hydro::apply / P_inv_hydro::apply with nothing left to the
    caller.  flow: capi.Flow with geometry, fiber operators and preconditioner, body operators and fiber links set;
    dense: capi.Dense holding stresslet_plus_complementary and M_inv, or None without a periphery."""

    def __init__(self, flow, dense, eta: float, device):
        import torch
        self.torch = torch
        self.flow, self.dense, self.eta = flow, dense, float(eta)
        self.n = flow.solution_size()
        kw = dict(dtype=torch.float64, device=device)
        self.res = torch.zeros(max(self.n, 1), **kw)
        self.y = torch.zeros(max(self.n, 1), **kw)
        self.launches = 0

    def _stream(self):
        return self.torch.cuda.current_stream().cuda_stream

    def apply(self, x):
        """System::apply_matvec (system.cpp:269-324): A x -- a view valid until the next call."""
        self.flow.apply_system_matvec_device(self.dense, x.data_ptr(), self.eta, self.res.data_ptr(), self._stream())
        self.launches = self.flow.stats()["launches"]
        return self.res[:self.n]

    def apply_preconditioner(self, x):
        """System::apply_preconditioner (system.cpp:248-262): P^-1 x -- a view valid until the next call."""
        self.flow.apply_system_preconditioner_device(self.dense, x.data_ptr(), self.y.data_ptr(), self._stream())
        return self.y[:self.n]

    def rhs(self, fiber_params, dt: float, f_external=None, body_forces=None, body_torques=None, v_growth=None,
            force_scale=None):
        """System::prep_state_for_solver's RHS (system.cpp:398-458), Solver::set_RHS's vector (solver_hydro.cpp:51-61):
        a new device tensor of solution_size().  fiber_params: the 7 per-fiber parameters of
        capi.Flow.build_fiber_operators (length_prev ... plus_hinged); f_external (N_f, 3), body_forces / body_torques
        (n_bodies, 3): device tensors or None (zero)."""
        torch = self.torch
        out = torch.empty(max(self.n, 1), dtype=torch.float64, device=self.res.device)
        p = lambda t: t.data_ptr() if t is not None and t.numel() else 0
        self.flow.build_system_rhs_device(*fiber_params, dt, self.eta, p(f_external), p(body_forces), p(body_torques),
                                          out.data_ptr(), v_growth=v_growth, force_scale=force_scale,
                                          stream=self._stream())
        self.launches = self.flow.stats()["launches"]
        return out[:self.n]

    def set_gmres(self, num_blocks: int = 300):
        """Size the solve's workspace (skb_flow_set_gmres) for up to num_blocks basis vectors per cycle."""
        self.flow.set_gmres(num_blocks)
        self._gmres_blocks = int(num_blocks)

    def solve(self, b, tol: float = 1e-10, num_blocks: int = 300, max_iters: int = 1000):
        """Solver::solve (solver_hydro.cpp:64-95): x = A^-1 b by restarted right-preconditioned GMRES on the device
        (skb_flow_solve_system_device), from x0 = 0.  b: a device tensor of solution_size().  Returns (x, info): x a new
        device tensor, info skb_solve_info as a dict plus "history", the implicit relative residual after each Arnoldi
        step.  The workspace is set up on first use, or again when num_blocks exceeds the one set up."""
        if getattr(self, "_gmres_blocks", 0) < num_blocks or self.flow.solution_size() != self.n:
            self.set_gmres(num_blocks)
        x = self.torch.empty(max(self.n, 1), dtype=self.torch.float64, device=self.res.device)
        info, hist = self.flow.solve_system_device(self.dense, b.data_ptr(), self.eta, x.data_ptr(), tol=tol,
                                                   num_blocks=num_blocks, max_iters=max_iters, stream=self._stream())
        self.launches = self.flow.stats()["launches"]
        return x[:self.n], dict(info, history=hist)


def iterate_system(op: SystemOperator, x, n_iter: int):
    """iterate() for whole solution vectors: `n_iter` times x <- A P^-1 x, rescaled to unit max-norm on the device."""
    for _ in range(n_iter):
        r = op.apply(op.apply_preconditioner(x))
        x = r / r.abs().max()
    return x

"""CPU calibration of the history bound of tests/test_gpu_solve_system.py (HISTORY_BOUND): the restatement
(tests/gmres_reference.py) run twice on each of its systems with system_reference.py's operators, once with numpy's dots
and once with the dots summed in the device kernels' blocked order; the worst difference of the implicit relative
residuals, step by step, must stay below a tenth of the bound, and both runs must take the same steps."""
import numpy as np
import pytest

import gmres_reference as gr
import system_reference as sr
from test_gpu_solve_system import CALIBRATED, ETA, HISTORY_BOUND, TOL, solve_case


@pytest.mark.parametrize("name,seed,shape,num_blocks", CALIBRATED)
def test_the_history_bound_is_ten_times_the_summation_order_difference(name, seed, shape, num_blocks):
    fib, shell, bodies, ops, links, x = solve_case(name, seed, shape=shape)
    ns = shell["pos"].shape[0]
    A = lambda v: sr.system_apply_matvec(fib, shell, bodies, ops, links, shell["M"], v, ETA)[0]
    P = lambda v: sr.system_apply_preconditioner(ops["A"], ops["n_nodes"], shell["Minv"] if ns else None, bodies["A"],
                                                 bodies["n_nodes"], v)
    b = A(x)
    _, numpy_dots = gr.gmres(A, P, b, tol=TOL, num_blocks=num_blocks)
    _, blocked = gr.gmres(A, P, b, tol=TOL, num_blocks=num_blocks, dot=gr.blocked_dot)
    assert numpy_dots["converged"] and blocked["converged"]
    assert numpy_dots["iterations"] == blocked["iterations"]
    d = np.abs(numpy_dots["history"] - blocked["history"]).max()
    print(f"\n{name}, {num_blocks} blocks: {numpy_dots['iterations']} steps, worst difference {d:.2e}")
    assert d <= HISTORY_BOUND / 10, d

"""GPU parity test of fibers longer than 1024 nodes: the self term's kernel keeps a fiber's nodes and strengths in shared
memory (48 B per node), so such a fiber needs more than the default 48 KB of dynamic shared memory, which
skb_flow_set_fibers raises for the kernel that launches.  The fiber flow with its self term and the matvec are
checked against the oracle, tolerance <= 1e-12 relative (max-norm and l2)."""
import numpy as np
import pytest

import oracle as orc
import skellysim_b200 as skb
from test_gpu_flow import _check, ft_of, load, make_system

pytestmark = pytest.mark.gpu


def test_fibers_above_1024_nodes():
    fib, shell, body = make_system(61, 3, 300, 0, 0, nodes=(1100, 1500, 2000))
    assert max(fib["n_nodes"]) * 48 > 48 * 1024
    eta = 0.7
    r_all = np.concatenate([fib["pos"], shell["pos"]])
    with skb.Flow(0) as fl:
        load(fl, fib, shell, body)
        v = fl.fiber_flow(r_all, fib["forces"], eta, subtract_self=True)
        m = fl.matvec(fib["forces"], shell["density"], body["density"], ft_of(body), eta)
    _check(v, orc.fiber_flow(r_all, fib["pos"], fib["n_nodes"], fib["lengths"], fib["forces"], eta, True))
    _check(m, orc.matvec_flow(fib, shell, body, eta))

"""CPU restatement of the body block and the fiber-body links of System::apply_matvec / ::apply_preconditioner -- TEST
INFRASTRUCTURE ONLY.  Citations are `file:line` in the SkellySim tree.  Arrays follow oracle/oracle.py: a 3 x n Eigen
matrix is an (n, 3) array, the solution vector is [fibers (4 per node) | shell (3 per node) | bodies (3 n_b + 6 each)]
(get_solution_maps, system.cpp:69-92).

    kernels::stresslet_times_normal(_times_density)   kernels.cpp:264-334          stresslet_times_normal(_times_density)
    SphericalBody::update_singularity_subtraction_vecs body_spherical.cpp:168-181   singularity_vectors
    SphericalBody::update_K_matrix / update_preconditioner  :74-86, 104-126        body_operator
    SphericalBody::matvec (BodyContainer::matvec)     :39-63 (body_container.cpp:487-504)  body_matvec
    BodyContainer::calculate_link_conditions          body_container.cpp:171-267   link_conditions
    System::apply_matvec / ::apply_preconditioner     system.cpp:269-324, 248-262  system_apply_matvec / _preconditioner

Dicts: fib = dict(pos, n_nodes, lengths) (tests/test_gpu_flow.py make_system); ops = the fiber operators of
oracle.fiber_container_matvec plus D_2_0 / D_3_0 per node count; links = dict(body (n_fibers,), site (n_fibers, 3),
rigidity (n_fibers,)); bodies = dict(pos, normals, centers, n_nodes (per body), weights, ex, ey, ez)."""
import numpy as np

import oracle as orc

# defects a test of the links must catch: the sign of omega x site in v_fiber swapped; length_prev_ in place of length_
# in xsss (the fiber's previous length instead of the current one)
LINK_DEFECTS = ("omega_site_sign", "xsss_length_prev")


def stresslet_times_normal(r, normals, reg=5e-3, epsilon_distance=1e-5):
    """(3N, 3N): block (i, j) = -3/(4 pi) (dr . n_j) dr dr^T / |dr|^5, dr = r_i - r_j, zero diagonal blocks
    (kernels.cpp:264-290; eta is unused there)."""
    r, normals = np.asarray(r, dtype=np.float64), np.asarray(normals, dtype=np.float64)
    N = r.shape[0]
    dr = r[:, None, :] - r[None, :, :]
    rn = np.linalg.norm(dr, axis=2)
    rn = np.where(rn < epsilon_distance, np.sqrt(rn * rn + reg * reg), rn)
    np.fill_diagonal(rn, 1.0)
    coeff = (-3.0 / (4.0 * np.pi)) * np.einsum("ijk,jk->ij", dr, normals) / rn**5
    np.fill_diagonal(coeff, 0.0)
    S = coeff[:, :, None, None] * dr[:, :, :, None] * dr[:, :, None, :]
    return S.transpose(0, 2, 1, 3).reshape(3 * N, 3 * N)


def stresslet_times_normal_times_density(r, normals, density, reg=5e-3, epsilon_distance=1e-5):
    """(N, 3): row i = -3/(4 pi) sum_{j != i} (dr . rho_j)(dr . n_j) dr / |dr|^5 (kernels.cpp:307-334)."""
    r, normals, density = (np.asarray(a, dtype=np.float64) for a in (r, normals, density))
    dr = r[:, None, :] - r[None, :, :]
    rn = np.linalg.norm(dr, axis=2)
    rn = np.where(rn < epsilon_distance, np.sqrt(rn * rn + reg * reg), rn)
    np.fill_diagonal(rn, 1.0)
    f0 = np.einsum("ijk,jk->ij", dr, density) * np.einsum("ijk,jk->ij", dr, normals) / rn**5
    np.fill_diagonal(f0, 0.0)
    return (-3.0 / (4.0 * np.pi)) * np.einsum("ij,ijk->ik", f0, dr)


def singularity_vectors(r, normals, weights):
    """ex_, ey_, ez_ of one body (N, 3) each: the stresslet contracted with the weights along x, y, z (:168-181)."""
    out = []
    for k in range(3):
        e = np.zeros((len(weights), 3))
        e[:, k] = weights
        out.append(stresslet_times_normal_times_density(r, normals, e))
    return out


def body_operator(r, normals, center, weights, ex, ey, ez):
    """A_ of one body as update_preconditioner assembles it (:104-126), with K_ of update_K_matrix (:74-86)."""
    n = r.shape[0]
    A = np.zeros((3 * n + 6, 3 * n + 6))
    A[:3 * n, :3 * n] = stresslet_times_normal(r, normals)
    for i in range(n):
        A[3 * i:3 * i + 3, 3 * i + 0] -= ex[i] / weights[i]
        A[3 * i:3 * i + 3, 3 * i + 1] -= ey[i] / weights[i]
        A[3 * i:3 * i + 3, 3 * i + 2] -= ez[i] / weights[i]
    K = np.zeros((3 * n, 6))
    for i in range(n):
        v = r[i] - center
        K[3 * i:3 * i + 3, 0:3] = np.eye(3)
        K[3 * i + 0, 3:6] = (0.0, v[2], -v[1])
        K[3 * i + 1, 3:6] = (-v[2], 0.0, v[0])
        K[3 * i + 2, 3:6] = (v[1], -v[0], 0.0)
    A[:3 * n, 3 * n:] = -K
    A[3 * n:, :3 * n] = -K.T
    A[3 * n:, 3 * n:] = np.eye(6)
    return A


def _body_offsets(n_nodes):
    n_nodes = np.asarray(n_nodes, dtype=np.int64)
    node_off = np.concatenate([[0], np.cumsum(n_nodes)])
    sol_off = np.concatenate([[0], np.cumsum(3 * n_nodes + 6)])
    return node_off, sol_off


def body_matvec(bodies, v_bodies, x_bodies):
    """BodyContainer::matvec (body_container.cpp:487-504) -> SphericalBody::matvec (body_spherical.cpp:39-63) per body:
    res_nodes = -(cx + cy + cz) - K U + v, res_com = -K^T lambda + U."""
    node_off, sol_off = _body_offsets(bodies["n_nodes"])
    res = np.empty(int(sol_off[-1]))
    for b, n in enumerate(bodies["n_nodes"]):
        a, s = int(node_off[b]), int(sol_off[b])
        d = x_bodies[s:s + 3 * n].reshape(n, 3)
        U = x_bodies[s + 3 * n:s + 3 * n + 6]
        w = bodies["weights"][a:a + n, None]
        c = (d[:, 0:1] / w) * bodies["ex"][a:a + n] + (d[:, 1:2] / w) * bodies["ey"][a:a + n] + \
            (d[:, 2:3] / w) * bodies["ez"][a:a + n]
        rr = bodies["pos"][a:a + n] - bodies["centers"][b]
        KU = U[:3] + np.cross(U[3:], rr)
        res[s:s + 3 * n] = (-c - KU + v_bodies[a:a + n]).reshape(-1)
        KTl = np.concatenate([d.sum(axis=0), np.cross(rr, d).sum(axis=0)])
        res[s + 3 * n:s + 3 * n + 6] = -KTl + U
    return res


def link_conditions(fib, ops, links, bodies, x_fibers, x_bodies, literal=False, defect=None):
    """BodyContainer::calculate_link_conditions (body_container.cpp:171-267).  Returns (velocities_on_fiber
    (n_fibers, 7), body_forces_torques (n_bodies, 6)).

    literal=False: every bound fiber reads its own slice of x_fibers and writes its own row (the evident intent).
    literal=True: the code as written -- `continue` for a free fiber skips `i_fib++` and `xt_offset += 4 n`
    (:202-204, 262-263), so after the first free fiber the bound ones read and write their neighbours' places.
    ops["length_prev"] is read by the "xsss_length_prev" defect only."""
    assert defect is None or defect in LINK_DEFECTS, defect
    n_nodes = [int(n) for n in fib["n_nodes"]]
    nfib, nb = len(n_nodes), len(bodies["n_nodes"])
    _, sol_off = _body_offsets(bodies["n_nodes"])
    vel = np.zeros((nfib, 7))
    ft = np.zeros((nb, 6))
    fib_off = np.concatenate([[0], np.cumsum(n_nodes)]).astype(int)
    xt_offset, i_fib = 0, 0
    for f, n in enumerate(n_nodes):
        i_body = int(links["body"][f])
        if i_body < 0:
            continue
        xo, col = (xt_offset, i_fib) if literal else (4 * fib_off[f], f)
        site_pos = np.asarray(links["site"][f], dtype=np.float64) - bodies["centers"][i_body]   # :209
        x_new = np.stack([x_fibers[xo + k * n:xo + (k + 1) * n] for k in range(3)])              # :210-213
        T0 = x_fibers[xo + 3 * n]                                                                # :215
        xs0 = ops["xs"][fib_off[f]]                                                              # :217
        L = fib["lengths"][f]
        L3 = ops["length_prev"][f] if defect == "xsss_length_prev" else L
        xss0 = ((2.0 / L) ** 2 * (x_new @ ops["D_2_0"][n]))[:, 0]                                # :218,220
        xsss0 = ((2.0 / L3) ** 3 * (x_new @ ops["D_3_0"][n]))[:, 0]                              # :219,221
        E = links["rigidity"][f]
        F = -E * xsss0 + xs0 * T0                                                                # :226
        Lb = -E * np.cross(site_pos, xsss0) + np.cross(site_pos, xs0) * T0 + E * np.cross(xs0, xss0)  # :231-237
        ft[i_body, :3] += F
        ft[i_body, 3:] += Lb
        s = int(sol_off[i_body]) + 3 * int(bodies["n_nodes"][i_body])
        U, w = x_bodies[s:s + 3], x_bodies[s + 3:s + 6]                                          # :184-194, 245-246
        sign = 1.0 if defect == "omega_site_sign" else -1.0
        vel[col, :3] = -U + sign * np.cross(w, site_pos)                                         # :249
        vel[col, 3] = -xs0 @ U + np.cross(xs0, site_pos) @ w                                     # :252
        vel[col, 4:] = np.cross(site_pos / np.linalg.norm(site_pos), w)                          # :256
        i_fib += 1
        xt_offset += 4 * n
    return vel, ft


def split(x, n_fib_nodes, n_shell):
    return x[:4 * n_fib_nodes], x[4 * n_fib_nodes:4 * n_fib_nodes + 3 * n_shell], x[4 * n_fib_nodes + 3 * n_shell:]


def system_apply_matvec(fib, shell, bodies, ops, links, M, x, eta, literal=False):
    """System::apply_matvec (system.cpp:269-324): returns (res, velocities_on_fiber, body_forces_torques).
    shell = dict(pos, normals); M = stresslet_plus_complementary_ (3 N_s, 3 N_s) or None without periphery."""
    nf, ns = int(np.sum(fib["n_nodes"])), shell["pos"].shape[0]
    x_f, x_s, x_b = split(np.asarray(x, dtype=np.float64), nf, ns)
    n_bodies = len(bodies["n_nodes"])
    node_off, sol_off = _body_offsets(bodies["n_nodes"])
    if n_bodies:
        vel, ft = link_conditions(fib, ops, links, bodies, x_f, x_b, literal)
    else:
        vel, ft = np.zeros((len(fib["n_nodes"]), 7)), np.zeros((0, 6))
    dens = np.concatenate([x_b[sol_off[b]:sol_off[b] + 3 * n].reshape(n, 3)
                           for b, n in enumerate(bodies["n_nodes"])]) if n_bodies else np.zeros((0, 3))
    body = dict(pos=bodies["pos"], normals=bodies["normals"], density=dens, centers=bodies["centers"],
                forces=ft[:, :3], torques=ft[:, 3:])
    res_f, v_all = orc.apply_matvec_fibers(fib, dict(shell, density=x_s.reshape(ns, 3)), body, ops, x_f, eta,
                                           vel if len(fib["n_nodes"]) else None)
    res_s = M @ x_s + v_all[nf:nf + ns].reshape(-1) if ns else np.zeros(0)                     # system.cpp:319
    res_b = body_matvec(bodies, v_all[nf + ns:], x_b) if n_bodies else np.zeros(0)              # system.cpp:320
    return np.concatenate([res_f, res_s, res_b]), vel, ft


def system_apply_preconditioner(fiber_A, n_fib_nodes, M_inv, body_A, body_n_nodes, x):
    """System::apply_preconditioner (system.cpp:248-262): A_LU_.solve per fiber, M_inv_ x_shell, A_LU_.solve per body
    (LAPACK's partial-pivoting solve here)."""
    nf = int(np.sum(n_fib_nodes))
    ns = 0 if M_inv is None else M_inv.shape[0] // 3
    x_f, x_s, x_b = split(np.asarray(x, dtype=np.float64), nf, ns)
    y_f = orc.fiber_apply_preconditioner(fiber_A, x_f, n_fib_nodes)
    y_s = M_inv @ x_s if ns else np.zeros(0)
    _, sol_off = _body_offsets(body_n_nodes)
    y_b = np.concatenate([np.linalg.solve(A, x_b[sol_off[b]:sol_off[b + 1]]) for b, A in enumerate(body_A)]) \
        if len(body_A) else np.zeros(0)
    return np.concatenate([y_f, y_s, y_b])

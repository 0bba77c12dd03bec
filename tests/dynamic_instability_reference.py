"""Restatement of System::dynamic_instability (dynamic_instability.cpp:25-194) as skb_flow_dynamic_instability runs it
(DESIGN.md §3.11): the Philox4x32-10 stream of skellysim_b200/csrc/philox.cuh, the catastrophe, growth, Poisson count
and site picks, and the nucleated fibers' straight lines, in the device's rounding order.  Python floats are IEEE
doubles and math.exp is the host's libm exp, so every value here is bitwise the library's."""
import math

import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF
CATASTROPHE, POISSON, PICK = 0, 1, 2
CHUNK = 256.0  # the largest mean of one Poisson inversion


def philox4x32_10(ctr, key):
    c0, c1, c2, c3 = (int(v) & MASK for v in ctr)
    k0, k1 = (int(v) & MASK for v in key)
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & MASK, (p0 >> 32) ^ c3 ^ k1, p0 & MASK
    return c0, c1, c2, c3


def uniform(seed, call, i, purpose):
    w = philox4x32_10((i, purpose, call & MASK, call >> 32), (seed & MASK, seed >> 32))
    return float(((w[1] << 32) | w[0]) >> 11) * 2.0 ** -53


def poisson(mu, seed, call):
    """the count: inversion in ceil(mu / 256) equal chunks, chunk i from draw (i, POISSON)"""
    if not mu > 0:
        return 0
    n_chunks = math.ceil(mu / CHUNK)
    m = mu / n_chunks
    cap = m + 40.0 * math.sqrt(m) + 40.0
    total = 0
    for c in range(n_chunks):
        u = uniform(seed, call, c, POISSON)
        k, p = 0, math.exp(-m)
        F = p
        while u > F and k < cap:
            k += 1
            p *= m / k
            F += p
        total += k
    return total


def rotation(q):
    """Eigen's toRotationMatrix, in the order of skb::quaternion_rotation"""
    w, x, y, z = (float(v) for v in q)
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [[1.0 - (tyy + tzz), txy - twz, txz + twy], [txy + twz, 1.0 - (txx + tzz), tyz - twx],
            [txz - twy, tyz + twx, 1.0 - (txx + tyy)]]


def straight_fiber(c, q, s_ref, n, L):
    """the nucleated fiber's nodes: origin = c + R(q) s_ref, u = (origin - c) / sqrt(|origin - c|^2),
    x_i = origin + u s_i, s_i = i (L / (n - 1)) and s_{n-1} = L (Eigen 3.4's LinSpaced)"""
    R = rotation(q)
    c = [float(v) for v in c]
    s = [float(v) for v in s_ref]
    o = [c[k] + ((R[k][0] * s[0] + R[k][1] * s[1]) + R[k][2] * s[2]) for k in range(3)]
    d = [o[k] - c[k] for k in range(3)]
    nrm = math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
    u = [d[k] / nrm for k in range(3)]
    step = L / (n - 1)
    x = np.empty((n, 3))
    for i in range(n):
        si = L if i == n - 1 else i * step
        for k in range(3):
            x[i, k] = o[k] + u[k] * si
    return x


DEFAULTS = dict(penalty_param=500.0, beta_tstep=1.0)


def dynamic_instability(di, dt, seed, call, lengths, params, binding, plus_pinned, sites_per_body, site_ref,
                        centers, quats, n_nodes_in=None, r_fib=None):
    """One call.  di: dict of skb_dynamic_instability; lengths, params (structured FIBER_PARAMS_DTYPE array), binding
    ((n, 2) int (body, site), -1 free), plus_pinned per fiber; sites_per_body and site_ref ((total, 3)) the bodies' site
    tables; centers / quats the placement.  Returns a dict: n_nodes, lengths, params, binding, v_growth, origin,
    positions (when r_fib and n_nodes_in are given) and removed, nucleated, grown, mu."""
    n_in = len(lengths)
    lengths = np.asarray(lengths, dtype=np.float64)
    binding = np.asarray(binding, dtype=np.int64).reshape(n_in, 2)
    if di["n_nodes"] == 0:
        out = dict(lengths=lengths.copy(), params=params.copy(), binding=binding.copy(), v_growth=None,
                   origin=np.arange(n_in), removed=0, nucleated=0, grown=0, mu=0.0)
        if n_nodes_in is not None:
            out["n_nodes"] = np.asarray(n_nodes_in).copy()
            out["positions"] = None if r_fib is None else np.asarray(r_fib).copy()
        return out
    off = np.concatenate([[0], np.cumsum(sites_per_body)]).astype(np.int64)
    n_sites = int(off[-1])
    thr = (math.exp(-dt * di["f_catastrophe"]),
           math.exp(-dt * (di["f_catastrophe"] * di["f_catastrophe_collision_scale"])))
    vel = (di["v_growth"], di["v_growth"] * di["v_grow_collision_scale"])
    occupied = np.zeros(n_sites, dtype=bool)
    n_active_old = 0
    keep, new_len, v_out = [], [], []
    for f in range(n_in):
        pinned = 1 if plus_pinned[f] else 0
        bound = binding[f, 0] >= 0
        n_active_old += bound
        if uniform(seed, call, f, CATASTROPHE) > thr[pinned]:
            continue
        keep.append(f)
        v = vel[pinned]
        new_len.append(float(lengths[f]) + dt * v)
        v_out.append(v)
        if bound:
            occupied[off[binding[f, 0]] + binding[f, 1]] = True
    mu = dt * di["nucleation_rate"] * (n_sites - n_active_old)
    inactive = [i for i in range(n_sites) if not occupied[i]]
    M = len(inactive)
    n_new = min(poisson(mu, seed, call), M)
    for k in range(n_new):
        u = uniform(seed, call, k, PICK)
        j = k + min(int(math.floor(u * (M - k))), M - k - 1)
        inactive[k], inactive[j] = inactive[j], inactive[k]
    picks = inactive[:n_new]
    body_of = np.searchsorted(off, picks, side="right") - 1
    n_out = len(keep) + n_new
    p_out = np.zeros(n_out, dtype=params.dtype)
    p_out[:len(keep)] = params[keep]
    p_out["length_prev"][:len(keep)] = lengths[keep]
    L0 = di["min_length"]
    for name, v in (("length_prev", L0), ("bending_rigidity", di["bending_rigidity"]), ("radius", di["radius"]),
                    ("penalty_param", 500.0), ("beta_tstep", 1.0), ("minus_clamped", 1), ("plus_hinged", 0)):
        p_out[name][len(keep):] = v
    b_out = np.concatenate([binding[keep], np.stack([body_of, np.asarray(picks) - off[body_of]], axis=1)
                            if n_new else np.zeros((0, 2), dtype=np.int64)]).astype(np.int64)
    out = dict(lengths=np.array(new_len + [L0] * n_new), params=p_out, binding=b_out,
               v_growth=np.array(v_out + [0.0] * n_new), origin=np.array(keep + [-1] * n_new),
               removed=n_in - len(keep), nucleated=n_new, grown=len(keep), mu=mu, picks=picks)
    if n_nodes_in is not None:
        n_nodes_in = np.asarray(n_nodes_in)
        out["n_nodes"] = np.concatenate([n_nodes_in[keep], np.full(n_new, di["n_nodes"])]).astype(np.int64)
        if r_fib is not None:
            foff = np.concatenate([[0], np.cumsum(n_nodes_in)])
            parts = [np.asarray(r_fib)[foff[f]:foff[f + 1]] for f in keep]
            for k, flat in enumerate(picks):
                b = int(body_of[k])
                parts.append(straight_fiber(centers[b], quats[b], site_ref[flat], di["n_nodes"], L0))
            out["positions"] = np.concatenate(parts) if parts else np.zeros((0, 3))
    return out

"""One-rank-per-GPU sharding of the pair-kernel path (used by bench.py; CPU-testable with gloo).

Targets are independent (each u_t is a private sum over all sources; the reference already exploits this across
OpenMP threads, kernels.cpp:58-65), so targets AND sources are block-partitioned over ranks and the only exchange
is ONE all-gather of the source strengths per evaluation (SURVEY.md 8e).  Positions are all-gathered once per
timestep.  This module only moves strengths between ranks; it computes no velocities."""
from __future__ import annotations

from dataclasses import dataclass


def block_range(n: int, world: int, rank: int):
    """Contiguous block [b, e) of rank `rank` when n items are split into `world` blocks of ceil(n/world)."""
    chunk = -(-n // world) if world > 0 else n
    b = min(n, rank * chunk)
    e = min(n, (rank + 1) * chunk)
    return b, e


@dataclass
class RankPartition:
    n_src: int
    n_trg: int
    world: int
    rank: int

    @property
    def src_chunk(self) -> int:  # all-gather slot size (equal on every rank)
        return -(-self.n_src // self.world)

    @property
    def src_range(self):
        return block_range(self.n_src, self.world, self.rank)

    @property
    def trg_range(self):
        return block_range(self.n_trg, self.world, self.rank)

    @property
    def gathered_rows(self) -> int:
        return self.src_chunk * self.world


def allgather_strengths(gathered, mine, group=None):
    """In-place all-gather of this rank's strength slot into `gathered` ((world*src_chunk, d) tensor; `mine` must be
    the view gathered[rank*src_chunk:(rank+1)*src_chunk]).  NCCL on GPUs, gloo on CPU."""
    import torch.distributed as dist
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_gather_into_tensor(gathered, mine, group=group)
    return gathered


def sym_row_owner(block_row: int, n_parts: int) -> int:
    """Owner of block row I of the symmetric kernel's upper triangle (mirror of sym_row_owner in
    csrc/skb_sym.cu): serpentine over rows, so every rank gets the same mix of long and short rows."""
    k, m = divmod(block_row, n_parts)
    return n_parts - 1 - m if (k & 1) else m


def sym_block_pairs(n_blocks: int, part: int, n_parts: int):
    """(I, J) block pairs a rank evaluates in both directions: rows it owns of the strict upper triangle, plus its
    diagonal blocks (I, I)."""
    for i in range(n_blocks):
        if sym_row_owner(i, n_parts) != part:
            continue
        yield i, i
        for j in range(i + 1, n_blocks):
            yield i, j


def reference_counts(n: int, world: int):
    """Block sizes of the reference's MPI decompositions: n // world each, the first n % world ranks one more
    (fibers: fiber_container_finite_difference.cpp:102-108; periphery nodes: periphery.cpp:387-400)."""
    return [n // world + (1 if r < n % world else 0) for r in range(world)]


def reference_rank_ranges(n_fibers: int, n_shell_nodes: int, n_body_nodes: int, rank: int, world: int):
    """The rows of [fibers | shell | bodies] one MPI rank of the reference owns, as the six arguments of
    skb_flow_set_target_ranges: whole fibers [f0, f1), periphery nodes [s0, s1), and all body nodes on rank 0
    (body_container.cpp keeps the bodies on world_rank_ 0)."""
    def block(n):
        c = reference_counts(n, world)
        b = sum(c[:rank])
        return b, b + c[rank]
    f0, f1 = block(n_fibers)
    s0, s1 = block(n_shell_nodes)
    b0, b1 = (0, n_body_nodes) if rank == 0 else (0, 0)
    return f0, f1, s0, s1, b0, b1


def system_rows(partition, fiber_n_nodes, n_shell: int, body_n_nodes):
    """The indices of the whole solution vector [fibers (4 per node) | shell (3 per node) | bodies (3 n + 6 each)] one
    member owns, ascending.  partition: its six target ranges (f0, f1, s0, s1, b0, b1), as skb_mflow_partition /
    capi.partition_query give them.  Besides its fibers' and periphery rows, the member owns the 3 rows of each body node
    in [b0, b1) and the six rows [U; w] of every body whose first node lies in [b0, b1) -- the rule of
    skb_mflow_apply_system_matvec."""
    import numpy as np
    f0, f1, s0, s1, b0, b1 = (int(v) for v in partition)
    fn = np.asarray(fiber_n_nodes, dtype=np.int64)
    node_off = np.concatenate([[0], np.cumsum(fn)])
    n_fib = int(node_off[-1])
    pieces = [np.arange(4 * node_off[f0], 4 * node_off[f1]), 4 * n_fib + np.arange(3 * s0, 3 * s1)]
    base, node = 4 * n_fib + 3 * int(n_shell), 0
    for n in (int(v) for v in body_n_nodes):
        lo, hi = max(b0, node), min(b1, node + n)
        if lo < hi:
            pieces.append(base + np.arange(3 * (lo - node), 3 * (hi - node)))
        if b0 <= node < b1:
            pieces.append(base + 3 * n + np.arange(6))
        node += n
        base += 3 * n + 6
    return np.concatenate(pieces).astype(np.int64)


def connect_group(flow, rank: int, world: int, group=None):
    """One rank per GPU: make `flow` (geometry and target ranges already set) a member of a peer-memory group.  Every
    rank exports the CUDA-IPC handle of its window, the 64-byte handles travel through torch.distributed once, every
    rank maps all peers' windows.  After this, flow.matvec_device / apply_matvec_device exchange strengths and partial
    velocities through NVLink loads / stores inside the library's own kernels -- no collective call per matvec."""
    import torch.distributed as dist
    flow.group_init(rank, world)
    if world == 1:
        return
    handles = [None] * world
    dist.all_gather_object(handles, flow.group_export(), group=group)
    for r in range(world):
        if r != rank:
            flow.group_import(r, handles[r])
    flow.group_warmup()  # every buffer at its final size before the first flag wait
    dist.barrier(group=group)


def allgatherv_rows(local, counts, group=None):
    """All-gather of per-rank row blocks of unequal length (fw of the own fibers -> fw of all fibers): pads every
    block to max(counts) rows, one all_gather_into_tensor, returns the concatenation without the padding.
    `local` is a (counts[rank], d) tensor; NCCL on GPUs, gloo on CPU."""
    import torch
    import torch.distributed as dist
    world = len(counts)
    if world == 1 or not dist.is_initialized():
        return local
    m = max(counts)
    pad = torch.zeros((m,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[:local.shape[0]] = local
    out = torch.empty((world * m,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, pad, group=group)
    return torch.cat([out[r * m:r * m + counts[r]] for r in range(world)])


class RankApplyMatvec:
    """One rank of System::apply_matvec (system.cpp:269-324) in the reference's decomposition, one rank per GPU.

    The rank owns whole fibers, a block of periphery nodes and (rank 0) the bodies (`reference_rank_ranges`); it holds
    only its own part of the solution vector, like the reference's local vectors.  Per matvec:

        fw_own   = force_operator_ * x_own                         (device, own fibers)
        fw_all   = all-gather(fw_own);  x_shell_all = all-gather(x_shell_own);  body strengths broadcast from rank 0
        v_own    = flow matvec over [own fiber nodes | own shell rows | own body rows]   (device)
        res_own  = A_ x_own - P vT(v_own) + xs_vT + y_BC            (device, own fibers)

    `flow` is a capi.Flow (or anything with its *_device methods) that already holds the FULL geometry and, after
    `set_target_ranges(*self.ranges)`, the operators of the own fibers.  All arrays are torch tensors on the flow's
    device; nothing is copied to the host.  This class only moves strengths between ranks and sequences the calls.
    """

    def __init__(self, flow, fiber_n_nodes, n_shell_nodes, n_body_nodes, n_bodies, rank, world, device="cpu",
                 group=None):
        import torch
        self.flow, self.rank, self.world, self.group = flow, rank, world, group
        self.torch = torch
        off = [0]
        for n in fiber_n_nodes:
            off.append(off[-1] + int(n))
        self.ranges_all = [reference_rank_ranges(len(fiber_n_nodes), n_shell_nodes, n_body_nodes, r, world)
                           for r in range(world)]
        self.ranges = self.ranges_all[rank]
        self.fib_counts = [off[r[1]] - off[r[0]] for r in self.ranges_all]       # fiber nodes per rank
        self.shell_counts = [r[3] - r[2] for r in self.ranges_all]
        self.n_fib, self.n_shell, self.n_body, self.n_bodies = off[-1], n_shell_nodes, n_body_nodes, n_bodies
        f0, f1, s0, s1, b0, b1 = self.ranges
        self.n_fib_own, self.n_shell_own, self.n_body_own = self.fib_counts[rank], s1 - s0, b1 - b0
        self.n_fibers_own = f1 - f0
        kw = dict(dtype=torch.float64, device=device)
        self._fw_own = torch.zeros((max(self.n_fib_own, 1), 3), **kw)
        self._fw_all = torch.zeros((max(self.n_fib, 1), 3), **kw)
        self._xs_all = torch.zeros((max(self.n_shell, 1), 3), **kw)
        self._v = torch.zeros((max(self.n_fib_own + self.n_shell_own + self.n_body_own, 1), 3), **kw)
        self._res = torch.zeros(max(4 * self.n_fib_own, 1), **kw)
        self._pads = {}
        for key, counts in (("fib", self.fib_counts), ("shell", self.shell_counts)):
            m = max(max(counts), 1)
            idx = torch.tensor([r * m + i for r in range(world) for i in range(counts[r])], dtype=torch.long,
                               device=device)
            self._pads[key] = (m, torch.zeros((m, 3), **kw), torch.zeros((world * m, 3), **kw), idx)

    def _gather(self, key, local, out):
        """all-gather of unequal row blocks into `out` (preallocated): pad -> all_gather_into_tensor -> index_select."""
        import torch.distributed as dist
        m, pad, gathered, idx = self._pads[key]
        if self.world == 1 or not dist.is_initialized():
            out[:local.shape[0]].copy_(local)
            return out
        pad[:local.shape[0]].copy_(local)
        dist.all_gather_into_tensor(gathered, pad, group=self.group)
        if idx.numel():
            self.torch.index_select(gathered, 0, idx, out=out[:idx.numel()])
        return out

    def _stream(self):
        t = self.torch
        return t.cuda.current_stream().cuda_stream if self._v.is_cuda else 0

    def apply(self, x_fib_own, x_shell_own, body_density, body_forces, body_torques, link_own, eta):
        """x_fib_own (4 n_fib_own,), x_shell_own (n_shell_own, 3), body_* as held by rank 0 ((n_body, 3), (n_bodies, 3)
        twice; other ranks pass buffers of the same shape to receive the broadcast), link_own (n_fibers_own, 7) or
        None.  Returns views (res_fib_own, v_shell_own, v_body_own) valid until the next call."""
        import torch.distributed as dist
        fl, st = self.flow, self._stream()
        if self.n_fib_own:
            fl.apply_fiber_force_device(x_fib_own.data_ptr(), self._fw_own.data_ptr(), st)
        self._gather("fib", self._fw_own[:self.n_fib_own], self._fw_all)
        self._gather("shell", x_shell_own, self._xs_all)
        if self.world > 1 and dist.is_initialized():
            for t in (body_density, body_forces, body_torques):
                if t.numel():
                    dist.broadcast(t, src=0, group=self.group)
        fl.matvec_device(self._fw_all.data_ptr(), self._xs_all.data_ptr(), body_density.data_ptr(),
                         body_forces.data_ptr(), body_torques.data_ptr(), float(eta), self._v.data_ptr(), st)
        if self.n_fib_own:
            fl.fiber_matvec_device(x_fib_own.data_ptr(), self._v.data_ptr(),
                                   link_own.data_ptr() if link_own is not None else 0, self._res.data_ptr(), st)
        a, b = self.n_fib_own, self.n_fib_own + self.n_shell_own
        return self._res[:4 * a], self._v[a:b], self._v[b:b + self.n_body_own]


class RankSystemOperator:
    """A and P^-1 of the whole mobility system, and its right-hand side, on ONE rank's local vector: the rank-per-GPU
    twin of solver_hydro.SystemOperator (A_fiber_hydro::apply / P_inv_hydro::apply / Solver::set_RHS of one MPI rank on
    its Tpetra local view).

    flow: a capi.Flow that is a connected group member (target ranges = `partition`, connect_group, fiber operators,
    group_set_body_operators, group_set_fiber_links); dense_matvec / dense_minv: capi.Dense on the flow's device holding
    the member's rows of stresslet_plus_complementary / M_inv (None without own periphery rows).  The local vector is
    x[local_rows] of the whole vector, local_rows = system_rows(partition, fiber_n_nodes, n_shell, body_n_nodes): the
    union over the ranks is the whole vector, each row once.  Every rank must make the same calls in the same order.
    This class sequences the calls and owns the work vectors; it computes nothing itself."""

    def __init__(self, flow, dense_matvec, dense_minv, partition, fiber_n_nodes, n_shell, body_n_nodes, eta, device):
        import torch
        self.torch = torch
        self.flow, self.dense_matvec, self.dense_minv, self.eta = flow, dense_matvec, dense_minv, float(eta)
        self.local_rows = system_rows(partition, fiber_n_nodes, n_shell, body_n_nodes)
        self.n = int(self.local_rows.size)
        kw = dict(dtype=torch.float64, device=device)
        self.res = torch.zeros(max(self.n, 1), **kw)
        self.y = torch.zeros(max(self.n, 1), **kw)
        self.b = torch.zeros(max(self.n, 1), **kw)  # owned: no call allocates while a peer may wait on a flag
        self.launches = 0

    def _stream(self):
        return self.torch.cuda.current_stream().cuda_stream

    @staticmethod
    def _ptr(t):
        return t.data_ptr() if t is not None and t.numel() else 0

    def apply(self, x_local):
        """the rank's rows of A x (System::apply_matvec) -- a view valid until the next call"""
        self.flow.group_apply_system_matvec_device(self.dense_matvec, self._ptr(x_local), self.eta, self.res.data_ptr(),
                                                   self._stream())
        self.launches = self.flow.stats()["launches"]
        return self.res[:self.n]

    def apply_preconditioner(self, x_local):
        """the rank's rows of P^-1 x (System::apply_preconditioner) -- a view valid until the next call"""
        self.flow.group_apply_system_preconditioner_device(self.dense_minv, self._ptr(x_local), self.y.data_ptr(),
                                                           self._stream())
        self.launches = self.flow.stats()["launches"]
        return self.y[:self.n]

    def rhs(self, fiber_params, dt: float, f_external=None, body_forces=None, body_torques=None, v_growth=None,
            force_scale=None):
        """the rank's rows of the RHS (System::prep_state_for_solver) -- a view valid until the next call.  fiber_params
        and v_growth / force_scale: of the OWN fibers; f_external (own fiber nodes, 3); body_forces / body_torques
        (n_bodies, 3) of ALL bodies, the same on every rank; None: zero."""
        self.flow.group_build_system_rhs_device(*fiber_params, dt, self.eta, self._ptr(f_external),
                                                self._ptr(body_forces), self._ptr(body_torques), self.b.data_ptr(),
                                                v_growth=v_growth, force_scale=force_scale, stream=self._stream())
        self.launches = self.flow.stats()["launches"]
        return self.b[:self.n]

    def set_gmres(self, num_blocks: int = 300):
        """Size the rank's solve workspace (skb_flow_set_gmres on its local rows) and the solution it returns.  A set-up
        call: it allocates, so every rank makes it before any rank's first solve (a peer on the same device may spin on
        a flag while another allocates)."""
        self.flow.set_gmres(num_blocks)
        self.x = self.torch.zeros_like(self.res)
        self._gmres_blocks = int(num_blocks)

    def solve(self, b_local, tol: float = 1e-10, num_blocks: int = 300, max_iters: int = 1000):
        """Solver::solve on the rank's local rows (skb_flow_group_solve_system_device): every rank calls it alike with
        its rows of b and gets its rows of x (a view valid until the next call) and info -- bitwise the same on every
        rank, history included.  Needs set_gmres(num_blocks or more) first."""
        if getattr(self, "_gmres_blocks", 0) < num_blocks:
            raise RuntimeError("RankSystemOperator.solve: call set_gmres(num_blocks) on every rank first")
        info, hist = self.flow.group_solve_system_device(self.dense_matvec, self.dense_minv, self._ptr(b_local),
                                                         self.eta, self.x.data_ptr(), tol=tol, num_blocks=num_blocks,
                                                         max_iters=max_iters, stream=self._stream())
        self.launches = self.flow.stats()["launches"]
        return self.x[:self.n], dict(info, history=hist)


class RankStepper:
    """System::step on one rank per GPU: the twin of timestep.Stepper for a capi.Flow that is a connected group member,
    with the same methods (positions, placement, step, backup, restore), so that timestep.run drives it unchanged.

    flow: the member (target ranges = `partition`, connect_group, fiber classes, group_set_body_frames or
    group_set_body_operators, a first group_place_bodies); dense: a capi.Dense on its device holding its row blocks of
    both periphery operators (None without own periphery rows).  params (the seven of Flow.build_fiber_operators),
    fiber_body, site_ref, v_growth and force_scale are given for ALL fibers, as to Stepper; the stepper keeps the own
    fibers' slices.  step's f_external is of ALL fiber nodes too.  Every member holds the whole geometry, so positions()
    and placement() are complete on every rank.  Every rank must make the same calls in the same order.

    The device buffers the step reads and writes are allocated here, once: no step or restore allocates through torch's
    allocator while a peer may wait on a flag (device: the flow's torch device).  After the step, x (the member's local rows of the solution,
    system_rows order) and tension (its own fiber nodes) hold the step's outputs."""

    def __init__(self, flow, dense, params, eta, partition, fiber_body=None, site_ref=None, v_growth=None,
                 force_scale=None, tol=1e-10, num_blocks=300, max_iters=1000, body_n_nodes=None, device="cuda"):
        import numpy as np
        import torch
        self.torch = torch
        self.flow, self.dense, self.eta = flow, dense, float(eta)
        self.tol, self.num_blocks, self.max_iters = tol, num_blocks, max_iters
        off = np.asarray(flow._fiber_off, dtype=np.int64)
        self.partition = tuple(int(v) for v in partition)
        f0, f1 = self.partition[:2]
        self.nodes = (int(off[f0]), int(off[f1]))  # the own fiber nodes [a, b)
        own = lambda v: v[f0:f1] if np.ndim(v) else v
        self.params = tuple(own(p) for p in params)
        self.fiber_body = None if fiber_body is None else np.asarray(fiber_body, dtype=np.int32).reshape(-1)[f0:f1]
        self.site_ref = None if site_ref is None else np.asarray(site_ref, dtype=np.float64).reshape(-1, 3)[f0:f1]
        self.v_growth, self.force_scale = own(v_growth), own(force_scale)
        body_n = getattr(flow, "_body_n", []) if body_n_nodes is None else body_n_nodes
        self.local_rows = system_rows(self.partition, np.diff(off), getattr(flow, "n_shell", 0), body_n)
        kw = dict(dtype=torch.float64, device=device)
        nb, m = int(flow.n_bodies), self.nodes[1] - self.nodes[0]
        self._fext = torch.zeros((max(m, 1), 3), **kw)
        self._force = torch.zeros((max(nb, 1), 3), **kw)
        self._torque = torch.zeros((max(nb, 1), 3), **kw)
        self._x = torch.zeros(max(int(self.local_rows.size), 1), **kw)
        self._tension = torch.zeros(max(m, 1), **kw)
        self._backup = None

    @property
    def x(self):
        return self._x[:self.local_rows.size]

    @property
    def tension(self):
        return self._tension[:self.nodes[1] - self.nodes[0]]

    def set_gmres(self, num_blocks=None):
        """skb_flow_set_gmres on the member's local rows: sizes the solve's workspace and everything the step uses.  A
        set-up call: every rank makes it before any rank's first step."""
        self.flow.set_gmres(int(self.num_blocks if num_blocks is None else num_blocks))

    def positions(self):
        return self.flow.fibers()

    def placement(self):
        import numpy as np
        if self.flow.n_bodies == 0:
            return np.zeros((0, 3)), np.zeros((0, 4))
        return self.flow.placement()

    def _stream(self):
        return self.torch.cuda.current_stream(self._x.device).cuda_stream if self._x.is_cuda else 0

    def _upload(self, dst, host):
        """host rows into the preallocated device buffer dst (no allocation on the device); returns its pointer"""
        import numpy as np
        if host is None or len(host) == 0:
            return 0
        dst[:len(host)].copy_(self.torch.from_numpy(np.ascontiguousarray(host, dtype=np.float64)))
        return dst.data_ptr()

    def step(self, dt, f_external=None, body_forces_torques=None):
        """one System::step on every member alike; returns the step's info, the same on every member (a NaN
        fiber_error: the solution was not finite and no member installed anything)"""
        import numpy as np
        a, b = self.nodes
        fe = None if f_external is None else np.asarray(f_external, dtype=np.float64).reshape(-1, 3)[a:b]
        ft = None if body_forces_torques is None else np.asarray(body_forces_torques, dtype=np.float64).reshape(-1, 6)
        p_fe = self._upload(self._fext, fe)
        p_f = self._upload(self._force, None if ft is None else ft[:, :3])
        p_t = self._upload(self._torque, None if ft is None else ft[:, 3:])
        return self.flow.group_step_device(*self.params, dt, self.eta, dense_matvec=self.dense, dense_minv=self.dense,
                                           d_f_external=p_fe, d_body_forces=p_f, d_body_torques=p_t,
                                           fiber_body=self.fiber_body, site_ref=self.site_ref,
                                           v_growth=self.v_growth, force_scale=self.force_scale, tol=self.tol,
                                           num_blocks=self.num_blocks, max_iters=self.max_iters,
                                           d_x_local=self._x.data_ptr() if self.local_rows.size else 0,
                                           d_tension=self._tension.data_ptr() if b > a else 0, stream=self._stream())

    def backup(self):
        self._backup = (self.positions(), *self.placement())

    def restore(self):
        """the backed-up geometry on this member: set_fibers and group_place_bodies, no group protocol"""
        import numpy as np
        r, c, q = self._backup
        self.flow.set_fibers(r, np.diff(self.flow._fiber_off), self.flow._lengths)
        if self.flow.n_bodies:
            self.flow.group_place_bodies(c, q)

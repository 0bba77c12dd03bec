"""world_size-2 gloo tests (CPU) of the N>1 sharding used by bench.py: block partition of sources and targets, one
all-gather of strengths, per-rank target blocks that tile the global result.  The pair sums themselves are evaluated
with the CPU oracle here (this is a test of the sharding logic, not of the CUDA kernels)."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, n_src, n_trg, out_dir):
    sys.path.insert(0, ROOT)
    import oracle as orc
    from skellysim_b200.distributed import RankPartition, allgather_strengths
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(5)  # identical global problem on every rank
    r_src, r_trg = rng.uniform(-1, 1, (n_src, 3)), rng.uniform(-1, 1, (n_trg, 3))
    f = rng.uniform(-1, 1, (n_src, 3))
    part = RankPartition(n_src, n_trg, world, rank)
    gathered = torch.zeros((part.gathered_rows, 3), dtype=torch.float64)
    mine = gathered[rank * part.src_chunk:(rank + 1) * part.src_chunk]
    b, e = part.src_range
    mine[:e - b] = torch.from_numpy(f[b:e])          # each rank only knows its own strengths
    allgather_strengths(gathered, mine)
    f_all = gathered.numpy()[:n_src]
    assert np.array_equal(f_all, f), "all-gather layout must reproduce the global strength array"
    tb, te = part.trg_range
    u_block = orc.stokeslet_direct(r_src, f_all, r_trg[tb:te])
    np.save(os.path.join(out_dir, f"u_{rank}.npy"), u_block)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("n_src,n_trg", [(64, 50), (33, 7), (5, 1)])
def test_two_rank_sharding_tiles_the_global_result(tmp_path, n_src, n_trg):
    import oracle as orc
    world = 2
    port = _free_port()
    mp.spawn(_worker, args=(world, port, n_src, n_trg, str(tmp_path)), nprocs=world, join=True)
    rng = np.random.default_rng(5)
    r_src, r_trg = rng.uniform(-1, 1, (n_src, 3)), rng.uniform(-1, 1, (n_trg, 3))
    f = rng.uniform(-1, 1, (n_src, 3))
    ref = orc.stokeslet_direct(r_src, f, r_trg)
    got = np.concatenate([np.load(tmp_path / f"u_{r}.npy") for r in range(world)])
    assert got.shape == ref.shape
    assert np.array_equal(got, ref)


def test_block_range_covers_everything():
    from skellysim_b200.distributed import block_range
    for n in (0, 1, 7, 8, 9, 1000):
        for world in (1, 2, 3, 4, 8):
            cover = []
            for r in range(world):
                b, e = block_range(n, world, r)
                assert 0 <= b <= e <= n
                cover += list(range(b, e))
            assert cover == list(range(n))


def _sym_worker(rank, world, port, n, block, out_dir):
    sys.path.insert(0, ROOT)
    import oracle as orc
    from skellysim_b200.distributed import sym_block_pairs
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(9)
    r = rng.uniform(-1, 1, (n, 3))
    f = rng.uniform(-1, 1, (n, 3))
    nb = -(-n // block)
    part = np.zeros((n, 3))
    # each rank: its block rows, both directions of every (I, J) pair from ONE geometry pass (here: two oracle calls)
    for i, j in sym_block_pairs(nb, rank, world):
        si, sj = slice(i * block, min(n, (i + 1) * block)), slice(j * block, min(n, (j + 1) * block))
        part[si] += orc.stokeslet_direct(r[sj], f[sj], r[si])        # forward: u_I += G f_J
        if i != j:
            part[sj] += orc.stokeslet_direct(r[si], f[si], r[sj])    # reverse: u_J += G f_I
    t = torch.from_numpy(part)
    dist.all_reduce(t)                                                # the one reduction of the symmetric layout
    if rank == 0:
        np.save(os.path.join(out_dir, "u_sym.npy"), t.numpy())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_symmetric_row_partition_reduces_to_the_full_self_interaction(tmp_path, world):
    import oracle as orc
    n, block = 300, 32
    mp.spawn(_sym_worker, args=(world, _free_port(), n, block, str(tmp_path)), nprocs=world, join=True)
    rng = np.random.default_rng(9)
    r = rng.uniform(-1, 1, (n, 3))
    f = rng.uniform(-1, 1, (n, 3))
    ref = orc.stokeslet_direct(r, f, r)
    got = np.load(tmp_path / "u_sym.npy")
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-13


def test_sym_row_owner_is_balanced_and_complete():
    from skellysim_b200.distributed import sym_block_pairs, sym_row_owner
    for nb in (1, 2, 7, 64, 177):
        for parts in (1, 2, 4, 8):
            owners = [sym_row_owner(i, parts) for i in range(nb)]
            assert all(0 <= o < parts for o in owners)
            seen = set()
            load = [0] * parts
            for p in range(parts):
                for i, j in sym_block_pairs(nb, p, parts):
                    assert (i, j) not in seen and i <= j
                    seen.add((i, j))
                    load[p] += 1
            assert len(seen) == nb * (nb + 1) // 2          # every unordered block pair exactly once
            if nb >= 8 * parts:
                assert max(load) - min(load) <= 0.05 * max(load) + parts


# ---- the reference's own rank decomposition (whole fibers | periphery nodes | bodies on rank 0) for the full
# ---- apply_matvec with per-fiber operators (SURVEY.md §8f N2): skb_flow_set_target_ranges + allgatherv of fw

def _small_system(seed=3, n_fibers=5):
    rng = np.random.default_rng(seed)
    n_nodes = [int(n) for n in rng.choice([4, 6, 8], size=n_fibers)]
    pos = []
    for n in n_nodes:
        x0, d = rng.uniform(-2, 2, 3), rng.normal(size=3)
        pos.append(x0 + np.linspace(0, 1, n)[:, None] * d / np.linalg.norm(d))
    fib = dict(pos=np.concatenate(pos), n_nodes=n_nodes, lengths=[1.0] * n_fibers)
    d = rng.normal(size=(31, 3))
    d /= np.linalg.norm(d, axis=1)[:, None]
    shell = dict(pos=6 * d, normals=-d, density=rng.normal(size=(31, 3)))
    e = rng.normal(size=(10, 3))
    e /= np.linalg.norm(e, axis=1)[:, None]
    body = dict(pos=0.3 * e, normals=e, density=rng.normal(size=(10, 3)), centers=np.zeros((1, 3)),
                forces=rng.normal(size=(1, 3)), torques=rng.normal(size=(1, 3)))
    ops = dict(n_nodes=n_nodes, A=[], force=[], D_1_0={}, P={}, length_prev=[], plus=[])
    xs = []
    for n in n_nodes:
        ops["A"].append(rng.normal(size=(4 * n, 4 * n)))
        ops["force"].append(rng.normal(size=(3 * n, 4 * n)))
        xs.append(rng.normal(size=(n, 3)))
        ops["length_prev"].append(1.0)
        ops["plus"].append(int(rng.integers(0, 2)))
        ops["D_1_0"].setdefault(n, rng.normal(size=(n, n)))
        ops["P"].setdefault(n, rng.normal(size=(4 * n - 14, 4 * n)))
    ops["xs"] = np.concatenate(xs)
    x = rng.normal(size=4 * sum(n_nodes))
    link = rng.normal(size=(n_fibers, 7))
    return fib, shell, body, ops, x, link


def _rank_matvec_worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    import oracle as orc
    from skellysim_b200.distributed import allgatherv_rows, reference_rank_ranges
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    fib, shell, body, ops, x, link = _small_system()
    n_nodes = ops["n_nodes"]
    off = np.concatenate([[0], np.cumsum(n_nodes)])
    nf, ns, nb = off[-1], shell["pos"].shape[0], body["pos"].shape[0]
    ranges = [reference_rank_ranges(len(n_nodes), ns, nb, r, world) for r in range(world)]
    f0, f1, s0, s1, b0, b1 = ranges[rank]
    # own fibers: fw_own = force_operator_ * x_own, then the exchange the reference does inside fc.flow
    x_own = x[4 * off[f0]:4 * off[f1]]
    fw_own = orc.apply_fiber_force(ops["force"][f0:f1], x_own, n_nodes[f0:f1])
    counts = [int(off[r[1]] - off[r[0]]) for r in ranges]
    fw_all = allgatherv_rows(torch.from_numpy(fw_own), counts).numpy()
    assert np.array_equal(fw_all, orc.apply_fiber_force(ops["force"], x, n_nodes))
    # the rank's rows of v_all (every rank evaluates only its own targets; sliced from the full oracle result here)
    v_all = orc.matvec_flow(dict(fib, forces=fw_all), shell, body, 0.9)
    v_own = np.concatenate([v_all[off[f0]:off[f1]], v_all[nf + s0:nf + s1], v_all[nf + ns + b0:nf + ns + b1]])
    own = dict(ops, n_nodes=n_nodes[f0:f1], A=ops["A"][f0:f1], xs=ops["xs"][off[f0]:off[f1]],
               length_prev=ops["length_prev"][f0:f1], plus=ops["plus"][f0:f1])
    res_own = orc.fiber_container_matvec(own, x_own, v_own[:off[f1] - off[f0]], link[f0:f1])
    np.savez(os.path.join(out_dir, f"rank_{rank}.npz"), res=res_own, v=v_own, ranges=np.array(ranges[rank]))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_reference_rank_decomposition_tiles_apply_matvec(tmp_path, world):
    import oracle as orc
    from skellysim_b200.distributed import reference_counts, reference_rank_ranges
    assert reference_counts(7, 3) == [3, 2, 2] and reference_counts(2, 4) == [1, 1, 0, 0]
    assert reference_rank_ranges(5, 31, 10, 0, 2) == (0, 3, 0, 16, 0, 10)
    assert reference_rank_ranges(5, 31, 10, 1, 2) == (3, 5, 16, 31, 0, 0)
    port = _free_port()
    mp.spawn(_rank_matvec_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    fib, shell, body, ops, x, link = _small_system()
    ref_res, ref_v = orc.apply_matvec_fibers(fib, shell, body, ops, x, 0.9, link)
    nf, ns = fib["pos"].shape[0], shell["pos"].shape[0]
    parts = [np.load(tmp_path / f"rank_{r}.npz") for r in range(world)]
    assert np.array_equal(np.concatenate([p["res"] for p in parts]), ref_res)
    # fiber, shell and body pieces of every rank tile v_all
    off = np.concatenate([[0], np.cumsum(ops["n_nodes"])])
    v_f, v_s, v_b = [], [], []
    for p in parts:
        f0, f1, s0, s1, b0, b1 = p["ranges"]
        nfo, nso = off[f1] - off[f0], s1 - s0
        v_f.append(p["v"][:nfo])
        v_s.append(p["v"][nfo:nfo + nso])
        v_b.append(p["v"][nfo + nso:])
    assert np.array_equal(np.concatenate(v_f + v_s + v_b), ref_v)


# ---- RankApplyMatvec: the sequencing + collectives of one rank's apply_matvec, with a stand-in for capi.Flow whose
# ---- *_device methods read/write the same raw addresses but compute with the CPU oracle (no GPU here)

class _FakeFlow:
    def __init__(self, fib, shell, body, ops, ranges):
        import ctypes
        self.C, self.fib, self.shell, self.body, self.ops = ctypes, fib, shell, body, ops
        self.off = np.concatenate([[0], np.cumsum(ops["n_nodes"])])
        self.f0, self.f1, self.s0, self.s1, self.b0, self.b1 = ranges
        self.calls = []

    def _view(self, ptr, n):
        return np.ctypeslib.as_array((self.C.c_double * n).from_address(ptr))

    def _own(self):
        o, f0, f1 = self.ops, self.f0, self.f1
        return dict(o, n_nodes=o["n_nodes"][f0:f1], A=o["A"][f0:f1], force=o["force"][f0:f1],
                    xs=o["xs"][self.off[f0]:self.off[f1]], length_prev=o["length_prev"][f0:f1], plus=o["plus"][f0:f1])

    def apply_fiber_force_device(self, px, pfw, stream):
        import oracle as orc
        own = self._own()
        n = int(self.off[self.f1] - self.off[self.f0])
        self._view(pfw, 3 * n)[:] = orc.apply_fiber_force(own["force"], self._view(px, 4 * n), own["n_nodes"]).reshape(-1)
        self.calls.append("force")

    def matvec_device(self, pff, psd, pbd, pf, pt, eta, pv, stream):
        import oracle as orc
        nf, ns, nb = int(self.off[-1]), self.shell["pos"].shape[0], self.body["pos"].shape[0]
        fib = dict(self.fib, forces=self._view(pff, 3 * nf).reshape(nf, 3).copy())
        shell = dict(self.shell, density=self._view(psd, 3 * ns).reshape(ns, 3).copy())
        body = dict(self.body, density=self._view(pbd, 3 * nb).reshape(nb, 3).copy(),
                    forces=self._view(pf, 3).reshape(1, 3).copy(), torques=self._view(pt, 3).reshape(1, 3).copy())
        v = orc.matvec_flow(fib, shell, body, eta)
        a, b = self.off[self.f0], self.off[self.f1]
        own = np.concatenate([v[a:b], v[nf + self.s0:nf + self.s1], v[nf + ns + self.b0:nf + ns + self.b1]])
        self._view(pv, own.size)[:] = own.reshape(-1)
        self.calls.append("flow")

    def fiber_matvec_device(self, px, pv, plink, pres, stream):
        import oracle as orc
        own = self._own()
        n = int(self.off[self.f1] - self.off[self.f0])
        link = self._view(plink, 7 * (self.f1 - self.f0)).reshape(-1, 7) if plink else None
        self._view(pres, 4 * n)[:] = orc.fiber_container_matvec(own, self._view(px, 4 * n),
                                                                self._view(pv, 3 * n).reshape(n, 3), link)
        self.calls.append("fiber_matvec")


def _rank_apply_worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    from skellysim_b200.distributed import RankApplyMatvec
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    fib, shell, body, ops, x, link = _small_system()
    ns, nb = shell["pos"].shape[0], body["pos"].shape[0]
    ram = RankApplyMatvec(None, ops["n_nodes"], ns, nb, 1, rank, world)
    ram.flow = _FakeFlow(fib, shell, body, ops, ram.ranges)
    off = np.concatenate([[0], np.cumsum(ops["n_nodes"])])
    f0, f1, s0, s1, b0, b1 = ram.ranges
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64))
    x_own = t(x[4 * off[f0]:4 * off[f1]])
    xs_own = t(shell["density"][s0:s1])
    # only rank 0 knows the body unknowns; the others pass receive buffers
    z = lambda a: t(a) if rank == 0 else torch.zeros(a.shape, dtype=torch.float64)
    bd, bf, bt = z(body["density"]), z(body["forces"]), z(body["torques"])
    link_own = t(link[f0:f1])
    for _ in range(2):  # twice: the preallocated buffers are reused
        res, v_s, v_b = ram.apply(x_own, xs_own, bd, bf, bt, link_own, 0.9)
    assert ram.flow.calls[-3:] == ["force", "flow", "fiber_matvec"]
    np.savez(os.path.join(out_dir, f"ram_{rank}.npz"), res=res.numpy(), v_s=v_s.numpy(), v_b=v_b.numpy())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_rank_apply_matvec_sequencing_and_collectives(tmp_path, world):
    import oracle as orc
    port = _free_port()
    mp.spawn(_rank_apply_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    fib, shell, body, ops, x, link = _small_system()
    ref_res, ref_v = orc.apply_matvec_fibers(fib, shell, body, ops, x, 0.9, link)
    nf, ns = fib["pos"].shape[0], shell["pos"].shape[0]
    parts = [np.load(tmp_path / f"ram_{r}.npz") for r in range(world)]
    assert np.array_equal(np.concatenate([p["res"] for p in parts]), ref_res)
    assert np.array_equal(np.concatenate([p["v_s"] for p in parts]), ref_v[nf:nf + ns])
    assert np.array_equal(np.concatenate([p["v_b"] for p in parts]), ref_v[nf + ns:])


# ---- the peer-memory group protocol (skb_group.cu / matvec_core), emulated on CPU with gloo ---------------------------
def _group_worker(rank, world, port, n_fibers, n_shell, block, out_dir):
    """One group member: push (all-gather of the own strengths), partial fiber velocities from the member's serpentine
    block rows of the symmetric fiber-fiber interaction (both directions of every block pair + own diagonal blocks),
    complete sums on the own periphery rows, pull (sum of the members' partials on the own fiber rows)."""
    sys.path.insert(0, ROOT)
    import oracle as orc
    from skellysim_b200 import capi
    from skellysim_b200.distributed import sym_block_pairs
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rng = np.random.default_rng(11)
    n_nodes = rng.choice([8, 16, 24], size=n_fibers).astype(np.int32)
    off = np.concatenate([[0], np.cumsum(n_nodes)])
    nf = int(off[-1])
    r_fib, r_shell = rng.uniform(-1, 1, (nf, 3)), rng.uniform(-2, 2, (n_shell, 3))
    f = rng.uniform(-1, 1, (nf, 3))
    f0, f1, s0, s1, _, _ = capi.partition_query(n_nodes, n_shell, 0, world, rank)
    a, b = int(off[f0]), int(off[f1])
    # PUSH: every member contributes the strengths of its own fibers only
    pieces = [None] * world
    dist.all_gather_object(pieces, (a, f[a:b]))
    f_all = np.zeros((nf, 3))
    for (pa, pf) in pieces:
        f_all[pa:pa + pf.shape[0]] = pf
    assert np.array_equal(f_all, f)
    # partial sums over the member's block rows (both directions), blocks of `block` nodes
    nb = -(-nf // block)
    blk = lambda i: slice(i * block, min(nf, (i + 1) * block))
    u_part = np.zeros((nf, 3))
    for (i, j) in sym_block_pairs(nb, rank, world):
        u_part[blk(i)] += orc.stokeslet_direct(r_fib[blk(j)], f_all[blk(j)], r_fib[blk(i)])
        if j != i:
            u_part[blk(j)] += orc.stokeslet_direct(r_fib[blk(i)], f_all[blk(i)], r_fib[blk(j)])
    v_shell_own = orc.stokeslet_direct(r_fib, f_all, r_shell[s0:s1])         # remainder rows: complete on the owner
    # PULL: own fiber rows = sum over the members' partials
    t = torch.from_numpy(u_part)
    dist.all_reduce(t)
    np.save(os.path.join(out_dir, f"g_{rank}.npy"), np.concatenate([t.numpy()[a:b], v_shell_own]))
    np.save(os.path.join(out_dir, f"r_{rank}.npy"), np.array([a, b, s0, s1]))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world,n_fibers,n_shell,block", [(2, 9, 21, 32), (3, 14, 5, 16), (2, 3, 0, 64)])
def test_group_protocol_tiles_the_global_result(tmp_path, world, n_fibers, n_shell, block):
    import oracle as orc
    port = _free_port()
    mp.spawn(_group_worker, args=(world, port, n_fibers, n_shell, block, str(tmp_path)), nprocs=world, join=True)
    rng = np.random.default_rng(11)
    n_nodes = rng.choice([8, 16, 24], size=n_fibers).astype(np.int32)
    nf = int(n_nodes.sum())
    r_fib, r_shell = rng.uniform(-1, 1, (nf, 3)), rng.uniform(-2, 2, (n_shell, 3))
    f = rng.uniform(-1, 1, (nf, 3))
    ref = orc.stokeslet_direct(r_fib, f, np.concatenate([r_fib, r_shell]))
    fib_rows, shell_rows = [], []
    for r in range(world):
        a, b, s0, s1 = np.load(tmp_path / f"r_{r}.npy")
        got = np.load(tmp_path / f"g_{r}.npy")
        want = np.concatenate([ref[a:b], ref[nf + s0:nf + s1]])
        assert got.shape == want.shape
        assert np.abs(got - want).max() <= 1e-12 * np.abs(ref).max()
        fib_rows.append((a, b))
        shell_rows.append((s0, s1))
    assert fib_rows[0][0] == 0 and fib_rows[-1][1] == nf and shell_rows[-1][1] == n_shell
    for (x, y) in zip(fib_rows, fib_rows[1:]):
        assert x[1] == y[0]

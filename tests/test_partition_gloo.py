"""world_size-2 CPU (gloo) test of the multi-rank design: a block partition of the tets plus a SUM all-reduce of the
per-rank gradients / CSR values, and a MIN all-reduce of the per-rank step bounds, reproduce the single-process result."""
import os
import sys

import numpy as np
import torch.distributed as dist
import torch.multiprocessing as mp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle as orc
    from ipc_b200 import mesh as M
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    V, T = M.grid_tets(4, 3, 3)
    m = M.Mesh(V, T, energy=0)
    M.deform(m, 3)
    ia, ja = m.csr_pattern(1)
    tb, te = m.nT * rank // world, m.nT * (rank + 1) // world  # the context's partition rule (api_mesh.cu)
    sub = M.Mesh.__new__(M.Mesh)
    sub.__dict__.update(m.__dict__)
    sub.T, sub.nT = m.T[tb:te], te - tb
    sub.restTriInv, sub.vol, sub.mu, sub.lam = m.restTriInv[tb:te], m.vol[tb:te], m.mu[tb:te], m.lam[tb:te]
    o = orc.Elastic(sub)
    g = torch.from_numpy(o.gradient(0.5, 0))
    a = torch.from_numpy(o.hessian_csr(0.5, ia, ja, 1, 1, 0))
    p = np.random.default_rng(1).standard_normal(3 * m.nV) * m.avgEdgeLen
    step = torch.tensor([o.inversion_step(p, 0.2, 1.0)[0]], dtype=torch.float64)
    dist.all_reduce(g, op=dist.ReduceOp.SUM); dist.all_reduce(a, op=dist.ReduceOp.SUM); dist.all_reduce(step, op=dist.ReduceOp.MIN)
    if rank == 0:
        full = orc.Elastic(m)
        ok = (np.allclose(g.numpy(), full.gradient(0.5, 0), rtol=0, atol=1e-12 * np.abs(g.numpy()).max())
              and np.allclose(a.numpy(), full.hessian_csr(0.5, ia, ja, 1, 1, 0), rtol=0, atol=1e-12 * np.abs(a.numpy()).max())
              and float(step) == full.inversion_step(p, 0.2, 1.0)[0])
        q.put(ok)
    dist.destroy_process_group()


def test_tet_partition_allreduce_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, 29641, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
    assert q.get(timeout=5) is True


def _contact_worker(rank, world, port, q):
    """Contact stage under the context's partition rules (api_contact.cu / constraint.cu / ccd.cu): every rank keeps a contiguous share of the
    pair lists and of the CCD candidates; SUM of the barrier energy / gradient / CSR values and MIN of the step reproduce one rank."""
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle as orc
    from ipc_b200 import scenes
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    m, info = scenes.ball_pile(2, res=5, seed=5, height=2)
    s = orc.Surf(m)
    dHat, p, kappa = info["dHat"], info["p"], 1e8
    mm, pa, pe, cand = s.constraint_set(dHat, nthreads=2)
    ia, ja = m.csr_pattern(1, extra_pairs=[(a, b) for r in list(mm) + list(pa) for a in ([(-r[0] - 1) if r[0] < 0 else r[0]] + [x for x in r[1:] if x >= 0])
                                            for b in ([(-r[0] - 1) if r[0] < 0 else r[0]] + [x for x in r[1:] if x >= 0]) if a < b]
                       + [(a, b) for e in pe if e[0] >= 0 for a in list(m.SFEdges[e[0]]) + list(m.SFEdges[e[1]]) for b in list(m.SFEdges[e[0]]) + list(m.SFEdges[e[1]]) if a != b])

    def share(n):  # [n*rank/world, n*(rank+1)/world)
        return slice(n * rank // world, n * (rank + 1) // world)

    mm_l, pa_l, pe_l, cand_l = mm[share(len(mm))], pa[share(len(pa))], pe[share(len(pa))], cand[share(len(cand))]
    E = torch.tensor([s.barrier_energy(mm_l, pa_l, pe_l, dHat, kappa)[0]], dtype=torch.float64)
    g = torch.from_numpy(s.barrier_gradient(mm_l, pa_l, pe_l, dHat, kappa))
    a = torch.from_numpy(s.barrier_hessian_csr(mm_l, pa_l, pe_l, dHat, kappa, ia, ja, 1, 1, nthreads=2))
    evf, eee = orc.ti_error(s.V, m.nV, p)
    step = torch.tensor([orc.ccd_partial(s, p, cand_l, 1e-6, evf, eee, 1.0, 2)[0]], dtype=torch.float64)
    for t, op in ((E, dist.ReduceOp.SUM), (g, dist.ReduceOp.SUM), (a, dist.ReduceOp.SUM), (step, dist.ReduceOp.MIN)):
        dist.all_reduce(t, op=op)
    if rank == 0:
        E1 = s.barrier_energy(mm, pa, pe, dHat, kappa)[0]
        g1 = s.barrier_gradient(mm, pa, pe, dHat, kappa)
        a1 = s.barrier_hessian_csr(mm, pa, pe, dHat, kappa, ia, ja, 1, 1, nthreads=2)
        st1 = orc.ccd_partial(s, p, cand, 1e-6, evf, eee, 1.0, 2)[0]
        ok = (len(mm) > 10 and abs(float(E) - E1) <= 1e-12 * abs(E1) and np.abs(g.numpy() - g1).max() <= 1e-12 * np.abs(g1).max()
              and np.abs(a.numpy() - a1).max() <= 1e-12 * np.abs(a1).max() and float(step) == st1)  # the step is bit-exact: min is exact
        q.put(ok)
    dist.destroy_process_group()


def test_contact_partition_allreduce_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_contact_worker, args=(r, 2, 29643, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
    assert q.get(timeout=5) is True


def _row_owner_worker(rank, world, port, q):
    """The row-owner rule (ipc_b200/partition.py = csrc/api_mesh.cu build_maps): every rank assembles the tets that touch its vertex range and
    keeps only the CSR rows (and gradient rows) it owns; the kept pieces are DISJOINT and their union is the single-process result -- no
    reduction of the Hessian, only a gather."""
    sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle as orc
    from ipc_b200 import mesh as M, partition as P
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    V, T = M.grid_tets(5, 4, 3)
    m = M.Mesh(V, T, energy=0)
    M.deform(m, 4)
    ia, ja = m.csr_pattern(1)
    b = P.vertex_boundaries(m.T, m.nV, world)
    vb, ve = b[rank], b[rank + 1]
    ids = P.assembled_tets(m.T, vb, ve)
    sub = M.Mesh.__new__(M.Mesh)
    sub.__dict__.update(m.__dict__)
    sub.T, sub.nT = m.T[ids], len(ids)
    sub.restTriInv, sub.vol, sub.mu, sub.lam = m.restTriInv[ids], m.vol[ids], m.mu[ids], m.lam[ids]
    o = orc.Elastic(sub)
    g = o.gradient(0.5, 0)
    a = o.hessian_csr(0.5, ia, ja, 1, 1, 0)
    a0, a1 = P.owned_value_range(ia, 1, vb, ve)
    g_own, a_own = np.zeros_like(g), np.zeros_like(a)
    g_own[3 * vb:3 * ve] = g[3 * vb:3 * ve]   # complete: every tet incident to an owned vertex was assembled here
    a_own[a0:a1] = a[a0:a1]
    tg, ta = torch.from_numpy(g_own), torch.from_numpy(a_own)
    dist.all_reduce(tg, op=dist.ReduceOp.SUM); dist.all_reduce(ta, op=dist.ReduceOp.SUM)  # disjoint supports: this is a gather
    cover = torch.zeros(world + 1, dtype=torch.int64); cover[rank] = len(ids); cover[world] = a1 - a0
    dist.all_reduce(cover, op=dist.ReduceOp.SUM)
    if rank == 0:
        full = orc.Elastic(m)
        ok = (np.allclose(tg.numpy(), full.gradient(0.5, 0), rtol=0, atol=1e-13 * np.abs(tg.numpy()).max())
              and np.allclose(ta.numpy(), full.hessian_csr(0.5, ia, ja, 1, 1, 0), rtol=0, atol=1e-13 * np.abs(ta.numpy()).max())
              and int(cover[world]) == ja.size                       # the owned value ranges tile the whole array
              and m.nT <= int(cover[:world].sum()) < 2 * m.nT)       # boundary tets are assembled twice, nothing is dropped
        q.put(ok)
    dist.destroy_process_group()


def test_row_owner_partition_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_row_owner_worker, args=(r, 2, 29643, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
    assert q.get(timeout=5) is True


def test_fused_energy_ownership_counts_every_tet_once_and_inside_the_assembled_set():
    """the rule of ipcgpu_elastic_energy_grad_hess on several ranks (kernels.h: ElasticArgs::e_row_lo / e_row_hi)"""
    from ipc_b200 import mesh as M, partition as P
    V, T = M.grid_tets(7, 6, 5)
    rng = np.random.default_rng(0)
    T = T[rng.permutation(len(T))]
    nV = len(V)
    for world in (1, 2, 3, 8):
        b = P.vertex_boundaries(T, nV, world)
        seen = np.zeros(len(T), dtype=int)
        for r in range(world):
            mine = P.energy_tets(T, b[r], b[r + 1])
            seen[mine] += 1
            assert np.isin(mine, P.assembled_tets(T, b[r], b[r + 1])).all()  # the rank that counts a tet also runs the kernel on it
        assert (seen == 1).all()

"""Launched by torchrun (one rank per GPU): the half-space stages with several ranks against the oracle (which equals the single-rank result,
tests/test_gpu_halfspace.py) -- replicated active / lagged sets and step bound, owner-summed energies and crossing counts in the host forms and
through ipcgpu_fetch_iteration's single collective, the rank-summed gradient and each rank's own Hessian rows.
   torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tests/mp/halfspace_check.py"""
import os
import struct
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch
import torch.distributed as dist

from ipc_b200 import lib as L
from test_gpu_halfspace import Small, nrel, oracle_all, rel, soa


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    sc = Small()
    m = sc.m
    ctx = L.Context(local)
    ids = [L.Context.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    ctx.comm_init(rank, world, ids[0])
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ia, ja = m.csr_pattern(1)
    ctx.set_csr(ia, ja, 1)
    ctx.set_state(soa(m.V))
    ctx.set_search_dir(sc.p)
    ctx.set_prev_state(soa(sc.Vprev))
    ctx.set_halfspaces(sc.origin, sc.normal, sc.vdt, sc.friction)
    ref = oracle_all(sc, m.V, ia, ja)
    part = ctx.partition_info()
    v0, v1 = part["row_vertex_begin"], part["row_vertex_end"]
    a0, a1 = part["value_begin"], part["value_end"]
    # host forms
    assert ctx.halfspace_constraint_set(sc.dHat) == len(ref["act"])
    act, _, _ = ctx.get_halfspace_sets()
    assert np.array_equal(act, ref["act"]), rank
    assert rel(ctx.halfspace_energy(sc.dHat, sc.kappa), ref["E"]) <= 1e-10
    alpha, rc = ctx.halfspace_step(None, 0.9, 1.0)
    assert rc == 0 and struct.pack("<d", alpha) == struct.pack("<d", ref["alpha"])
    assert ctx.halfspace_crossings() == ref["cross"]
    g = ctx.halfspace_gradient(sc.dHat, sc.kappa, np.zeros(3 * m.nV))
    assert nrel(g, ref["g"]) <= 1e-10
    a = ctx.halfspace_hessian(sc.dHat, sc.kappa, 1, np.zeros(ja.size))
    assert nrel(a[a0:a1], ref["a"][a0:a1]) <= 1e-9 or not ref["a"][a0:a1].any() and not a[a0:a1].any()
    assert ctx.halfspace_friction_lag(sc.dHat, sc.kappa) == len(ref["lag"])
    _, lag, lam = ctx.get_halfspace_sets()
    assert np.array_equal(lag, ref["lag"]) and nrel(lam, ref["lam"]) <= 1e-13
    assert rel(ctx.halfspace_friction_energy(sc.eps2), ref["Ef"]) <= 1e-10
    gf = ctx.halfspace_friction_gradient(sc.eps2, np.zeros(3 * m.nV))
    assert nrel(gf, ref["gf"]) <= 1e-10
    # deferred: the energies and the crossing count complete in the fetch's collective; the rows this rank owns hold its whole Hessian part
    ctx.halfspace_constraint_set(sc.dHat, want=False)
    ctx.halfspace_energy(sc.dHat, sc.kappa, want=False)
    ctx.halfspace_friction_energy(sc.eps2, want=False)
    ctx.halfspace_crossings(want=False)
    ctx.step_bound_set(1.0)
    ctx.halfspace_step(None, 0.9, None)
    ctx.csr_set_zero()
    ctx.halfspace_hessian(sc.dHat, sc.kappa, 1)
    ctx.halfspace_friction_hessian(sc.eps2, 1)
    it = ctx.fetch_iteration()
    assert it.status == 0 and it.n_halfspace_active == len(ref["act"]) and it.n_halfspace_crossings == ref["cross"]
    assert rel(it.energy_halfspace, ref["E"]) <= 1e-10 and rel(it.energy_halfspace_friction, ref["Ef"]) <= 1e-10
    assert struct.pack("<d", it.alpha_halfspace) == struct.pack("<d", ref["alpha"])
    a = ctx.download(L.BUF_CSR_VALUES, ja.size)
    want = (ref["a"] + ref["af"])[a0:a1]
    assert nrel(a[a0:a1], want) <= 1e-9 or not want.any() and not a[a0:a1].any()
    owned = [e for e in ref["act"] if v0 <= e[1] < v1]
    got = [None] * world
    dist.all_gather_object(got, len(owned))
    assert sum(got) == len(ref["act"])
    ctx.close()
    dist.barrier()
    if rank == 0:
        print(f"HALFSPACE_CHECK world={world} OK active={len(ref['act'])}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

"""Launched by torchrun (one rank per GPU): the device-built sparsity pattern is the same full pattern on every rank, equals the host mirror
of the global contact sets, and the owned value ranges tile [0, nnz).
   torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tests/mp/device_pattern_check.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch
import torch.distributed as dist

from bench import contact_pattern_pairs
from ipc_b200 import lib as L
from ipc_b200 import scenes


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    dHat = info["dHat"]
    ctx = L.Context(local)
    ids = [L.Context.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    ctx.comm_init(rank, world, ids[0])
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_state(m.V_soa)
    mm, pa, pe, _ = ctx.constraint_set(dHat, 1)  # replicated build: the global sets, for the host mirror
    ia_h, ja_h = m.csr_pattern(1, extra_pairs=contact_pattern_pairs(m, mm, pa, pe))
    ctx.enable_device_pattern(1)
    ctx.set_contact_partition(1)  # partitioned build + exchange: the pattern must come from the global lists
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.update_pattern(0, want=False)
    it = ctx.fetch_iteration()
    assert it.status == 0
    ia, ja = ctx.get_pattern()
    assert np.array_equal(ia, ia_h) and np.array_equal(ja, ja_h), rank
    part = ctx.partition_info()
    got = [None] * world
    dist.all_gather_object(got, (ia.tobytes(), ja.tobytes(), part["value_begin"], part["value_end"]))
    assert all(g[0] == got[0][0] and g[1] == got[0][1] for g in got)
    ranges = sorted((g[2], g[3]) for g in got)
    assert ranges[0][0] == 0 and ranges[-1][1] == ja.size and all(ranges[i][1] == ranges[i + 1][0] for i in range(world - 1)), ranges
    ctx.set_contact_partition(0)
    ctx.close()
    dist.barrier()
    if rank == 0:
        print(f"DEVICE_PATTERN_CHECK world={world} OK nnz={ja.size}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

"""Cost of the device-built sparsity pattern on C5 (146 x sphere1K.msh, 1M tets), device events throughout:
  1. ipcgpu_update_pattern eagerly, when the contact blocks are unchanged and when they change (states A and B alternate);
  2. the replayed Newton iteration (bench.py's device-resident chain) with the update stage against without it, both graphs alternated at
     the same state; and the graph with the stage when every replay changes the pattern;
  3. the host path the stage replaces -- this repository's host mirror, not the reference's std::set build: download of the contact sets,
     numpy csr_pattern + contact_pattern_pairs, ipcgpu_set_csr, and the offset search (ensure_offsets) the next Hessian call runs.
Prints one JSON line with the card's name, SM clock and power limit read in the same run.
    python profiles/device_pattern_timing.py [--reps 20]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from ipc_b200 import lib as L  # noqa: E402


DT2 = 0.025 ** 2


class Args:
    tets, res, scene = 1_000_000, 10, "c5"


def gpu_info():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,clocks.sm,clocks.max.sm,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except Exception as e:  # (reported, not fatal)
        return f"nvidia-smi unavailable: {e}"


def med(x):
    return float(np.median(x))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    m, info = bench.build_scene(Args())
    dHat, p, h = info["dHat"], info["p"], m.avgEdgeLen / 3
    ctx = L.Context(0)
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_state(m.V_soa)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    # state B: half of the feasible step along p (closer contact, another active set)
    ctx.constraint_set(dHat, 1, fetch=False)
    a = ctx.inversion_step(p, 0.2, 1.0)
    a = ctx.ccd_partial(None, bench.TI_TOL, evf, eee, a)
    a = ctx.hash_build_swept(None, a, h)
    a, _ = ctx.ccd_full(bench.TI_TOL, evf, eee, a)
    VA, VB = m.V_soa, np.ascontiguousarray((m.V + 0.5 * a * p.reshape(-1, 3)).T).ravel()
    out = {"gpu": gpu_info(), "scene": f"C5, {m.nT} tets, {m.nV} vertices", "reps": args.reps}

    # 3. host path (first: it leaves the context in host mode)
    t_dl, t_np, t_set, t_off = [], [], [], []
    ctx.set_canonical_order(1)
    for r in range(args.reps // 4 + 2):
        ctx.set_state(VB if r % 2 else VA)
        ctx.constraint_set(dHat, 1, fetch=False)
        ctx.sync()
        t0 = time.perf_counter()
        mm, pa, pe, _ = ctx.constraint_set(dHat, 1)  # (includes the set build; subtracted below)
        t1 = time.perf_counter()
        ctx.constraint_set(dHat, 1, fetch=False)
        t2 = time.perf_counter()
        ia, ja = m.csr_pattern(1, extra_pairs=bench.contact_pattern_pairs(m, mm, pa, pe))
        t3 = time.perf_counter()
        ctx.set_csr(ia, ja, 1)
        t4 = time.perf_counter()
        ctx.elastic_hessian(DT2, 1, 1, 1, None)  # ensure_offsets + the assembly
        ctx.sync()
        t5 = time.perf_counter()
        ctx.elastic_hessian(DT2, 1, 1, 1, None)  # the assembly alone
        ctx.sync()
        t6 = time.perf_counter()
        if r >= 2:
            t_dl.append((t1 - t0) - (t2 - t1))
            t_np.append(t3 - t2)
            t_set.append(t4 - t3)
            t_off.append((t5 - t4) - (t6 - t5))
    out["host_mirror_ms"] = {"download_sets": 1e3 * med(t_dl), "numpy_csr_pattern": 1e3 * med(t_np), "set_csr": 1e3 * med(t_set),
                             "ensure_offsets": 1e3 * med(t_off), "total": 1e3 * (med(t_dl) + med(t_np) + med(t_set) + med(t_off)), "nnz_A_B": None}

    # 1. eager update, unchanged / changed
    ctx.enable_device_pattern(1)
    ctx.set_canonical_order(0)
    nnz = {}
    t_ch, t_un = [], []
    for r in range(args.reps + 2):
        name = "B" if r % 2 else "A"
        ctx.set_state(VB if r % 2 else VA)
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.sync()
        ctx.timer_start(); ctx.update_pattern(want=False); tc = ctx.timer_stop()
        ch = ctx.pattern_info()
        ctx.timer_start(); ctx.update_pattern(want=False); tu = ctx.timer_stop()
        un = ctx.pattern_info()
        assert ch[0] == 1 and un[0] == 0, (ch, un)
        nnz[name] = ch[1]
        if r >= 2:
            t_ch.append(tc); t_un.append(tu)
    out["update_eager_ms"] = {"changed": med(t_ch), "unchanged": med(t_un), "changed_min_max": [min(t_ch), max(t_ch)], "unchanged_min_max": [min(t_un), max(t_un)]}
    out["host_mirror_ms"]["nnz_A_B"] = [nnz["A"], nnz["B"]]

    # 2. replayed iteration with / without the stage
    ctx.set_search_dir(p)

    def enqueue(stage):
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        if stage:
            ctx.update_pattern(want=False)
        ctx.elastic_energy_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.barrier_energy(dHat, bench.KAPPA, want=False)
        ctx.barrier_gradient(dHat, bench.KAPPA, None)
        ctx.barrier_hessian(dHat, bench.KAPPA, 1, None)
        ctx.step_bound_set(1.0)
        ctx.inversion_step(None, 0.2, None)
        ctx.ccd_partial(None, bench.TI_TOL, evf, eee, None)
        ctx.hash_build_swept(None, None, h)
        ctx.ccd_full(bench.TI_TOL, evf, eee, None)

    ctx.set_state(VA)
    graphs = {}
    for stage in (True, False):
        enqueue(stage)
        ctx.fetch_iteration()
        ctx.capture_begin()
        enqueue(stage)
        graphs[stage] = ctx.capture_end()
    for _ in range(3):
        for g in graphs.values():
            ctx.graph_launch(g)
    assert ctx.fetch_iteration().status == 0
    times = {True: [], False: []}
    for r in range(args.reps):
        for stage in ((True, False) if r % 2 else (False, True)):
            ctx.timer_start(); ctx.graph_launch(graphs[stage]); times[stage].append(ctx.timer_stop())
    assert ctx.fetch_iteration().status == 0
    t_chg = []
    for r in range(args.reps + 2):  # every replay after the first changes the pattern (A is in place already)
        ctx.set_state(VB if r % 2 else VA)
        ctx.timer_start(); ctx.graph_launch(graphs[True]); t = ctx.timer_stop()
        assert ctx.fetch_iteration().status == 0 and ctx.pattern_info()[0] == (1 if r else 0)
        if r >= 2:
            t_chg.append(t)
    out["replayed_iteration_ms"] = {"with_stage_unchanged": med(times[True]), "without_stage": med(times[False]), "with_stage_changed_every_replay": med(t_chg),
                                    "with_min_max": [min(times[True]), max(times[True])], "without_min_max": [min(times[False]), max(times[False])]}
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()

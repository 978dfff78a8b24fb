"""Cost the half-space stages add to a replayed C5 iteration (146 x sphere1K.msh, 1M tets) with a ground plane about 0.5 sqrt(dHat) below the
lowest vertex (the bottom balls have active vertices) and a downward component in p (the plane bound runs on moving vertices):
  1. the step-bound chain (step set, inversion filter, partial CCD, swept grid, full CCD) without and with ipcgpu_halfspace_step;
  2. the derivative chain (constraint set, elastic energy/gradient/Hessian, barrier terms) without and with the plane constraint set,
     energy, gradient and Hessian;
each captured once and replayed, the two forms alternated, device-event medians.  The line search with planes is not timed here.
Prints one JSON line with the card's name, SM clock and power limit read in the same run.
    python profiles/halfspace_timing.py [--reps 20]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import bench  # noqa: E402
from device_pattern_timing import Args, gpu_info, med  # noqa: E402
from ipc_b200 import lib as L  # noqa: E402

DT2 = 0.025 ** 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    m, info = bench.build_scene(Args())
    dHat, h, kappa, tol = info["dHat"], m.avgEdgeLen / 3, bench.KAPPA, bench.TI_TOL
    sq = np.sqrt(dHat)
    p = np.array(info["p"], dtype=np.float64).reshape(-1, 3)
    p[:, 1] -= 3.0 * sq
    p = np.ascontiguousarray(p).ravel()
    ctx = L.Context(0)
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_canonical_order(0)
    ctx.set_state(m.V_soa)
    ctx.set_search_dir(p)
    ctx.enable_device_pattern(1)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    ctx.set_halfspaces([[0.0, m.V[:, 1].min() - 0.5 * sq, 0.0]], [[0.0, 1.0, 0.0]], None, [0.0])
    n_act = ctx.halfspace_constraint_set(dHat)

    def step_chain(planes):
        ctx.step_bound_set(1.0)
        ctx.inversion_step(None, 0.2, None)
        if planes:
            ctx.halfspace_step(None, 0.9, None)
        ctx.ccd_partial(None, tol, evf, eee, None)
        ctx.hash_build_swept(None, None, h)
        ctx.ccd_full(tol, evf, eee, None)

    def deriv_chain(planes):
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        if planes:
            ctx.halfspace_constraint_set(dHat, want=False)
        ctx.update_pattern(want=False)
        ctx.elastic_energy_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.barrier_energy(dHat, kappa, want=False)
        ctx.barrier_gradient(dHat, kappa, None)
        ctx.barrier_hessian(dHat, kappa, 1, None)
        if planes:
            ctx.halfspace_energy(dHat, kappa, want=False)
            ctx.halfspace_gradient(dHat, kappa, None)
            ctx.halfspace_hessian(dHat, kappa, 1, None)

    out = {"gpu": gpu_info(), "scene": f"C5, {m.nT} tets, {m.nV} vertices", "reps": args.reps, "plane_active_entries": n_act}
    for name, chain in (("step_bound_chain", step_chain), ("derivative_chain", deriv_chain)):
        gids = {}
        for planes in (False, True):
            chain(planes)  # eager first: lazy allocations
            it = ctx.fetch_iteration()
            ctx.capture_begin()
            chain(planes)
            gids[planes] = ctx.capture_end()
            if name == "step_bound_chain":
                out[f"alpha_{'with' if planes else 'without'}_plane"] = it.alpha
        times = {False: [], True: []}
        for _ in range(args.reps):
            for planes in (False, True):
                ctx.set_state(m.V_soa)
                ctx.sync()
                ctx.timer_start()
                ctx.graph_launch(gids[planes])
                times[planes].append(ctx.timer_stop())
                ctx.fetch_iteration()
        out[name] = {"without_planes_ms": med(times[False]), "with_planes_ms": med(times[True]), "added_ms": med(times[True]) - med(times[False])}
        for g in gids.values():
            ctx.graph_destroy(g)
    out["line_search"] = "not measured"
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()

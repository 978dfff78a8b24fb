"""What the reproducible mode (ipcgpu_set_canonical_order(ctx, 2)) costs on C5 (146 x sphere1K.msh, 1M tets, ~8.8k contact pairs).
Two contexts, one at level 0 and one at level 2, each capture bench.py's iteration (constraint set, device-built pattern, elastic
energy / gradient / Hessian, barrier gradient and Hessian, inversion bound, partial CCD, swept grid, full CCD); the replays alternate between
them and are timed with device events on the context stream.  Also the eager time of the stages the mode changes (constraint set with its
sorts and indices, barrier gradient, barrier Hessian) and the launches per iteration.  Then the eager constraint set with the candidates
(wantCand = 1) at levels 0, 1 and 2, on C5 and on C3 (ball_on_mat, the ball lowered to half a contact distance over the mat), with the
largest bucket of the canonical order (entries of one list that share their first component).  Prints one JSON line with the card's name,
SM clock and power limit read in the same run.
    python profiles/reproducible_timing.py [--reps 30]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import bench  # noqa: E402
import numpy as np  # noqa: E402
from device_pattern_timing import Args, gpu_info, med  # noqa: E402
from ipc_b200 import lib as L  # noqa: E402
from ipc_b200 import scenes  # noqa: E402

DT2 = 0.025 ** 2
KAPPA = bench.KAPPA
TOL = 1e-6


def spread(t):
    return {"median": med(t), "min": min(t), "max": max(t)}


def largest_bucket(lists):
    return max((int(np.unique(a[:, 0], return_counts=True)[1].max()) for a in lists if len(a)), default=0)


def constraint_set_levels(m, dHat, reps):
    """eager constraint set with the candidates at levels 0, 1 and 2, alternated per repetition"""
    ctx = L.Context(0)
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_state(m.V_soa)
    t, launches = {0: [], 1: [], 2: []}, {}
    for r in range(reps + 2):
        for level in (0, 1, 2):
            ctx.set_canonical_order(level)
            n0 = ctx.launch_count()
            ctx.timer_start()
            ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
            dt = ctx.timer_stop()
            launches[level] = ctx.launch_count() - n0
            if r >= 2:
                t[level].append(dt)
    ctx.set_canonical_order(1)
    mm, pa, pe, cand = ctx.constraint_set(dHat, 1)
    ctx.close()
    return {"pairs": {"active": len(mm), "mollified": len(pa), "candidates": len(cand)}, "largest_bucket": largest_bucket((mm, pa, cand)),
            "ms": {f"level{k}": spread(v) for k, v in t.items()}, "launches": {f"level{k}": v for k, v in launches.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    m, info = bench.build_scene(Args())
    dHat = info["dHat"]
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, info["p"])
    h = m.avgEdgeLen / 3.0

    def iteration(ctx):
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.update_pattern(0, want=False)
        ctx.elastic_energy_grad_hess(DT2, 1, 1, 1)
        ctx.barrier_gradient(dHat, KAPPA, None)
        ctx.barrier_hessian(dHat, KAPPA, 1, None)
        ctx.step_bound_set(1.0)
        ctx.inversion_step(None, 0.2, None)
        ctx.ccd_partial(None, TOL, evf, eee, None)
        ctx.hash_build_swept(None, None, h)
        ctx.ccd_full(TOL, evf, eee, None)

    ctxs, gids, out = {}, {}, {"gpu": gpu_info(), "reps": args.reps}
    for level in (0, 2):
        ctx = L.Context(0)
        ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
        ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
        ctx.set_canonical_order(level)
        ctx.set_state(m.V_soa)
        ctx.set_search_dir(info["p"])
        ctx.enable_device_pattern(1)
        iteration(ctx)  # the eager run: lazy allocations
        ctx.fetch_iteration()
        ctx.capture_begin()
        iteration(ctx)
        gids[level] = ctx.capture_end()
        ctxs[level] = ctx
    nC, nP, _ = ctxs[2].constraint_set_sizes()
    out["scene"] = f"C5, {m.nT} tets, {m.nV} vertices, {nC} active + {nP} mollified pairs"
    replay = {0: [], 2: []}
    launches = {}
    for r in range(args.reps + 2):
        for level in (0, 2):
            ctx = ctxs[level]
            n0 = ctx.launch_count()
            ctx.timer_start()
            ctx.graph_launch(gids[level])
            t = ctx.timer_stop()
            launches[level] = ctx.launch_count() - n0
            ctx.fetch_iteration()
            if r >= 2:
                replay[level].append(t)
    out["replay_ms"] = {f"level{k}": spread(v) for k, v in replay.items()}
    out["launches_per_iteration"] = {f"level{k}": v for k, v in launches.items()}
    stages = {}
    for level in (0, 2):
        ctx = ctxs[level]
        t = {"constraint_set": [], "barrier_gradient": [], "barrier_hessian": []}
        for _ in range(args.reps):
            for name, fn in (("constraint_set", lambda: ctx.constraint_set(dHat, 1, fetch=False, sizes=False)),
                             ("barrier_gradient", lambda: ctx.barrier_gradient(dHat, KAPPA, None)),
                             ("barrier_hessian", lambda: ctx.barrier_hessian(dHat, KAPPA, 1, None))):
                ctx.timer_start()
                fn()
                t[name].append(ctx.timer_stop())
        ctx.fetch_iteration()
        stages[f"level{level}"] = {k: spread(v) for k, v in t.items()}
    out["eager_stage_ms"] = stages
    for level in (0, 2):
        ctxs[level].graph_destroy(gids[level])
        ctxs[level].close()
    mc, ic = scenes.ball_on_mat_c3()
    mc.V[ic["n_mat_verts"]:, 2] -= ic["gap"] - 0.5 * np.sqrt(ic["dHat"])
    out["eager_constraint_set_with_candidates"] = {"C5": constraint_set_levels(m, dHat, args.reps),
                                                   f"C3 ball_on_mat, {mc.nT} tets": constraint_set_levels(mc, ic["dHat"], args.reps)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()

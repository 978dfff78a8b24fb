"""Cost of capturing the device linear solves (the deferred form of ipcgpu_solve_pcg / _multilevel as conditional graph nodes), on C5
(146 x sphere1K.msh, 1M tets) and on a small contact scene (scenes.ball_on_mat(): a 40 x 40 mat and one ball), where launch and
synchronisation overhead weigh most:
  1. the solve alone: the synchronous call (host reads the residual test every 25 iterations) against one replay of a graph holding the
     deferred solve, alternating, both solvers, both to 1e-6;
  2. the whole Newton iteration with the multilevel solve (constraint set, device-built pattern, derivatives, solve, step bound with the CFL
     branch, line search) as ONE graph, against the same calls made eagerly;
  3. the first solve after a pattern change (the full-row structure is rebuilt on the device) against a solve on an unchanged pattern.
Medians of device-event and wall-clock times with their min / max.  Every repetition starts from the same state.  Prints one JSON line (and
writes it under profiles/results/ with --out) with the card's name, SM clock and power limit read in the same run.
    python profiles/solve_capture_timing.py [--reps 10] [--out profiles/results/solve_capture_timing_h100.json]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

import bench  # noqa: E402
from device_pattern_timing import Args, gpu_info, med  # noqa: E402
from ipc_b200 import lib as L  # noqa: E402
from ipc_b200 import scenes  # noqa: E402

DT2 = 0.025 ** 2
TOL_PCG = 1e-6


def stats(v):
    return {"device": med([t[0] for t in v]), "wall": med([t[1] for t in v]), "device_min_max": [min(t[0] for t in v), max(t[0] for t in v)],
            "wall_min_max": [min(t[1] for t in v), max(t[1] for t in v)]}


def run_scene(name, m, info, reps):
    dHat, h, kappa, tol = info["dHat"], m.avgEdgeLen / 3, bench.KAPPA, bench.TI_TOL
    ctx = L.Context(0)
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_canonical_order(0)
    ctx.set_state(m.V_soa)
    ctx.enable_device_pattern(1)
    xt = m.V.copy()  # one implicit-Euler step under gravity: the Newton direction is a descent direction of the line search's energy
    xt[:, 2] -= 9.81 * DT2
    ctx.set_xtilde(np.ascontiguousarray(xt.T).ravel())
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    terms = dict(elastic_coef=DT2, dHat=dHat, kappa=kappa, inertia=True)
    out = {"scene": f"{name}, {m.nT} tets, {m.nV} vertices", "reps": reps}

    def derivatives():
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.update_pattern(want=False)
        ctx.elastic_energy_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.barrier_gradient(dHat, kappa, None)
        ctx.barrier_hessian(dHat, kappa, 1, None)
        ctx.inertia_gradient(1, None)

    def iteration():
        derivatives()
        ctx.solve_pcg_multilevel(rel_tol=TOL_PCG, max_iter=5000, want_x=False, adopt=True, deferred=True)
        ctx.step_bound_set(1.0)
        ctx.inversion_step(None, 0.2, None)
        ctx.ccd_partial(None, tol, evf, eee, None)
        ctx.ccd_cfl(dHat, 1, h, tol, evf, eee, None)
        ctx.line_search(**terms)

    def timed(fn):
        ctx.sync()
        t0 = time.perf_counter()
        ctx.timer_start()
        fn()
        dev = ctx.timer_stop()
        return dev, 1e3 * (time.perf_counter() - t0)

    # 1. the solve alone on the system at the scene's state
    ctx.set_state(m.V_soa)
    derivatives()
    out["solve_ms"] = {}
    for sname, solve in (("block_jacobi", ctx.solve_pcg), ("multilevel", ctx.solve_pcg_multilevel)):
        solve(None, TOL_PCG, 5000, want_x=False, adopt=True)  # the eager run: lazy allocations
        ctx.capture_begin()
        solve(rel_tol=TOL_PCG, max_iter=5000, want_x=False, adopt=True, deferred=True)
        gid = ctx.capture_end()
        times = {"eager": [], "graph": []}
        its = {}
        for r in range(reps + 2):
            for form in (("eager", "graph") if r % 2 else ("graph", "eager")):
                t = timed((lambda: solve(None, TOL_PCG, 5000, want_x=False, adopt=True)) if form == "eager" else (lambda: ctx.graph_launch(gid)))
                s = ctx.solve_info()
                assert s.status == 0, s.status
                its[form] = s.iterations
                if r >= 2:
                    times[form].append(t)
        out["solve_ms"][sname] = {"iterations": its, **{f: stats(v) for f, v in times.items()}}
        ctx.graph_destroy(gid)

    # 2. the whole Newton iteration: one graph against the same calls made eagerly
    ctx.set_state(m.V_soa)
    iteration()
    ctx.fetch_iteration()
    ctx.set_state(m.V_soa)
    ctx.capture_begin()
    iteration()
    g_it = ctx.capture_end()
    times = {"eager": [], "graph": []}
    res = {}
    for r in range(reps + 2):
        for form in (("eager", "graph") if r % 2 else ("graph", "eager")):
            ctx.set_state(m.V_soa)
            t = timed(iteration if form == "eager" else (lambda: ctx.graph_launch(g_it)))
            s, sv, it = ctx.step_control_info(), ctx.solve_info(), ctx.fetch_iteration()
            assert s.status == 0 and sv.status == 0 and it.status == 0
            res[form] = {"alpha": s.alpha, "solve_iterations": sv.iterations}
            if r >= 2:
                times[form].append(t)
    out["iteration_ms"] = {"result": res, **{f: stats(v) for f, v in times.items()}}
    ctx.graph_destroy(g_it)

    # 3. the first solve after a pattern change against one on an unchanged pattern (synchronous multilevel calls)
    p = info["p"]  # (the second state: half of the feasible step along the scene's direction -- more contacts, another pattern)
    ctx.set_state(m.V_soa)
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    a = ctx.inversion_step(p, 0.2, 1.0)
    a = ctx.ccd_partial(None, tol, evf, eee, a)
    a = ctx.hash_build_swept(None, a, h)
    a, _ = ctx.ccd_full(tol, evf, eee, a)
    states = [m.V_soa, np.ascontiguousarray((m.V + 0.5 * a * p.reshape(-1, 3)).T).ravel()]
    times = {"changed": [], "unchanged": []}
    nnz = set()
    for r in range(reps + 2):
        for k in (0, 1):
            ctx.set_state(states[k])
            derivatives()
            changed, n_nz, _ = ctx.pattern_info()
            t_changed = timed(lambda: ctx.solve_pcg_multilevel(None, TOL_PCG, 5000, want_x=False))
            ctx.set_state(states[k])
            derivatives()
            assert ctx.pattern_info()[0] == 0
            t_same = timed(lambda: ctx.solve_pcg_multilevel(None, TOL_PCG, 5000, want_x=False))
            nnz.add(n_nz)
            if r >= 2 and changed:
                times["changed"].append(t_changed)
                times["unchanged"].append(t_same)
    out["pattern_change_solve_ms"] = {"nnz": sorted(nnz), **{f: stats(v) for f, v in times.items() if v}}
    ctx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = {"gpu": gpu_info(), "rel_tol": TOL_PCG}
    m, info = scenes.ball_on_mat()
    out["small"] = run_scene("ball_on_mat (40 x 40 mat, one ball)", m, info, args.reps)
    m, info = bench.build_scene(Args())
    out["c5"] = run_scene("C5", m, info, args.reps)
    out["gpu_after"] = gpu_info()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

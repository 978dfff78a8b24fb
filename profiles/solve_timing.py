"""Cost of the three built-in linear solvers on C5 (146 x sphere1K.msh, 1M tets) at the state and right-hand side of step_control_timing.py
(one implicit-Euler step under gravity, H p = -g on the device-resident matrix): block-Jacobi PCG (ipcgpu_solve_pcg), PCG with the
multilevel additive Schwarz preconditioner (ipcgpu_solve_pcg_multilevel) and PCG with smoothed-aggregation multigrid
(ipcgpu_solve_pcg_amg), alternating, all to 1e-6.  Per solver: iterations, the time of a
whole solve, the set-up (a solve limited to one iteration: hierarchy or block inverses, the start of the loop and that iteration) and the
time per iteration from the two, as device-event medians with min-max.  Prints one JSON line with the card's name, SM clock and power limit
read in the same run; no device setting is changed.
    python profiles/solve_timing.py [--reps 5]"""
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
TOL = 1e-6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    m, info = bench.build_scene(Args())
    dHat, kappa = info["dHat"], bench.KAPPA
    ctx = L.Context(0)
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_canonical_order(0)
    ctx.set_state(m.V_soa)
    ctx.enable_device_pattern(1)
    xt = m.V.copy()
    xt[:, 2] -= 9.81 * DT2
    ctx.set_xtilde(np.ascontiguousarray(xt.T).ravel())
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.update_pattern(want=False)
    ctx.elastic_energy_grad_hess(DT2, 1, 1, 1)
    ctx.barrier_gradient(dHat, kappa, None)
    ctx.barrier_hessian(dHat, kappa, 1, None)
    ctx.inertia_gradient(1, None)
    solvers = {"block_jacobi": ctx.solve_pcg, "multilevel": ctx.solve_pcg_multilevel, "amg": ctx.solve_pcg_amg}
    out = {"gpu": gpu_info(), "scene": f"C5, {m.nT} tets, {m.nV} vertices", "rel_tol": TOL, "reps": args.reps}

    def timed(solve, max_iter):
        ctx.sync()
        ctx.timer_start()
        _, it, res = solve(None, TOL, max_iter, want_x=False)
        return ctx.timer_stop(), it, res

    runs = {k: {"solve": [], "setup": []} for k in solvers}
    iters = {}
    for r in range(args.reps + 1):  # (the first repetition warms up: allocations, the full-row structure, module loads)
        for name in list(solvers)[r % 3:] + list(solvers)[:r % 3]:  # (each solver first in turn)
            t_all, it, res = timed(solvers[name], 20000)
            t_one, _, _ = timed(solvers[name], 1)
            assert res <= TOL, (name, it, res)
            iters[name] = it
            if r:
                runs[name]["solve"].append(t_all)
                runs[name]["setup"].append(t_one)
    for name, t in runs.items():
        per_it = [(a - b) / (iters[name] - 1) for a, b in zip(t["solve"], t["setup"])]
        out[name] = {"iterations": iters[name],
                     "solve_ms": {"median": med(t["solve"]), "min_max": [min(t["solve"]), max(t["solve"])]},
                     "setup_and_first_iteration_ms": {"median": med(t["setup"]), "min_max": [min(t["setup"]), max(t["setup"])]},
                     "ms_per_iteration": {"median": med(per_it), "min_max": [min(per_it), max(per_it)]}}
    domains, nbytes = ctx.multilevel_info()
    out["multilevel"]["domains_per_level"] = domains
    out["multilevel"]["inverse_bytes"] = nbytes
    out["amg"]["hierarchy"] = ctx.amg_info()
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()

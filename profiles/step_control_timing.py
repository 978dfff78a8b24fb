"""Cost of the step control on the device (ipcgpu_ccd_cfl_ti + ipcgpu_line_search) on C5 (146 x sphere1K.msh, 1M tets):
  1. the CFL branch and the line search, host-driven (eager: one synchronisation per decision) against one replay of the captured form
     (conditional graph nodes), device-event medians, wall-clock medians and the halvings of each loop;
  2. the whole Newton iteration (constraint set, derivative chain, step bound with the CFL branch, line search) as ONE graph against the
     two-part form a caller has without the feature: the iteration graph with the full CCD (bench.py's chain), a fetch, then the line
     search driven from the host.
Every repetition starts from the same state.  Prints one JSON line with the card's name, SM clock and power limit read in the same run.
    python profiles/step_control_timing.py [--reps 10]"""
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

DT2 = 0.025 ** 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    m, info = bench.build_scene(Args())
    dHat, h, kappa, tol = info["dHat"], m.avgEdgeLen / 3, bench.KAPPA, bench.TI_TOL
    ctx = L.Context(0)
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_canonical_order(0)
    ctx.set_state(m.V_soa)
    ctx.enable_device_pattern(1)
    # one implicit-Euler step under gravity: xTilta = x + dt^2 g, and the Newton direction H p = -g solved on the device (PCG), so that the line
    # search sees a descent direction (the scene's own p is a CCD stress direction, along which every trial raises the energy)
    xt = m.V.copy()
    xt[:, 2] -= 9.81 * DT2
    ctx.set_xtilde(np.ascontiguousarray(xt.T).ravel())
    ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
    ctx.update_pattern(want=False)
    ctx.elastic_energy_grad_hess(DT2, 1, 1, 1)
    ctx.barrier_gradient(dHat, kappa, None)
    ctx.barrier_hessian(dHat, kappa, 1, None)
    ctx.inertia_gradient(1, None)
    _, pcg_iters, pcg_res = ctx.solve_pcg(None, 1e-6, 5000, want_x=False, adopt=True)
    evf, eee = L.Context.ti_error(m.V_soa, m.nV, None)
    terms = dict(elastic_coef=DT2, dHat=dHat, kappa=kappa, inertia=True)
    out = {"gpu": gpu_info(), "scene": f"C5, {m.nT} tets, {m.nV} vertices", "reps": args.reps, "newton_direction_pcg": [pcg_iters, pcg_res]}

    def reset():
        ctx.set_state(m.V_soa)
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)

    def step_control():
        ctx.step_bound_set(1.0)
        ctx.inversion_step(None, 0.2, None)
        ctx.ccd_partial(None, tol, evf, eee, None)
        ctx.ccd_cfl(dHat, 1, h, tol, evf, eee, None)
        ctx.line_search(**terms)

    def derivatives():
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.update_pattern(want=False)
        ctx.elastic_energy_grad_hess(DT2, 1, 1, 1, None, None)
        ctx.barrier_energy(dHat, kappa, want=False)
        ctx.barrier_gradient(dHat, kappa, None)
        ctx.barrier_hessian(dHat, kappa, 1, None)

    def iteration_full_ccd():  # bench.py's chain
        derivatives()
        ctx.step_bound_set(1.0)
        ctx.inversion_step(None, 0.2, None)
        ctx.ccd_partial(None, tol, evf, eee, None)
        ctx.hash_build_swept(None, None, h)
        ctx.ccd_full(tol, evf, eee, None)

    def whole_iteration():
        derivatives()
        step_control()

    def timed(fn):
        ctx.sync()
        t0 = time.perf_counter()
        ctx.timer_start()
        fn()
        dev = ctx.timer_stop()
        return dev, 1e3 * (time.perf_counter() - t0)

    # 1. eager against one replay
    reset(); step_control(); ctx.fetch_iteration()
    reset(); ctx.capture_begin(); step_control(); g_sc = ctx.capture_end()
    times = {"eager": [], "graph": []}
    sc = {}
    for r in range(args.reps + 2):
        for form in (("eager", "graph") if r % 2 else ("graph", "eager")):
            reset()
            t = timed(step_control if form == "eager" else (lambda: ctx.graph_launch(g_sc)))
            s = ctx.step_control_info()
            assert s.status == 0, s.status
            sc[form] = dict(alpha=s.alpha, alpha_cfl=s.alpha_cfl, full_ccd=s.full_ccd, halvings=[s.halvings_inversion, s.halvings_intersection, s.halvings_armijo,
                                                                                                  s.halvings_post_check], post_check_rebuilt=s.post_check_rebuilt)
            if r >= 2:
                times[form].append(t)
    assert sc["eager"] == sc["graph"], sc
    out["step_control"] = sc["eager"]
    out["cfl_and_line_search_ms"] = {f: {"device": med([t[0] for t in v]), "wall": med([t[1] for t in v]), "device_min_max": [min(t[0] for t in v), max(t[0] for t in v)]}
                                     for f, v in times.items()}

    # 2. the whole iteration as one graph against the two-part form
    reset(); whole_iteration(); ctx.fetch_iteration()
    reset(); iteration_full_ccd(); ctx.fetch_iteration()
    reset(); ctx.capture_begin(); whole_iteration(); g_one = ctx.capture_end()
    reset(); ctx.capture_begin(); iteration_full_ccd(); g_two = ctx.capture_end()

    def two_part():
        ctx.graph_launch(g_two)
        ctx.fetch_iteration()
        ctx.line_search(**terms)

    def one_graph():
        ctx.graph_launch(g_one)
        ctx.fetch_iteration()

    times = {"one_graph": [], "two_part": []}
    for r in range(args.reps + 2):
        for form in (("one_graph", "two_part") if r % 2 else ("two_part", "one_graph")):
            ctx.set_state(m.V_soa)
            t = timed(one_graph if form == "one_graph" else two_part)
            assert ctx.step_control_info().status == 0
            if r >= 2:
                times[form].append(t)
    out["iteration_ms"] = {f: {"device": med([t[0] for t in v]), "wall": med([t[1] for t in v]), "device_min_max": [min(t[0] for t in v), max(t[0] for t in v)]}
                           for f, v in times.items()}
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()

"""Cost of the point-in-tetrahedron half of ipcgpu_intersection_free on C5 (146 x sphere1K.msh, 1M tets) with a cloud of 10^5 codimension-0
points in the pile's box: the check without points (vCoDim all 3) and with them, each captured once and replayed, the two forms alternated,
device-event medians.  The difference is the point-in-tetrahedron stage (grid, sort and scan).  Prints one JSON line with the card's name, SM
clock and power limit read in the same run.
    python profiles/codim_timing.py [--reps 30] [--points 100000]"""
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
from ipc_b200 import codim, lib as L  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--points", type=int, default=100_000)
    args = ap.parse_args()
    m0, _ = bench.build_scene(Args())
    rng = np.random.default_rng(3)
    lo, hi = m0.V.min(0), m0.V.max(0)
    P = lo + (hi - lo) * rng.uniform(0.0, 1.0, (args.points, 3))
    m = codim.codim_scene([dict(codim=3, V=m0.V_rest, T=m0.T, SF=m0.SF), dict(codim=0, V=P)], energy=m0.energy)
    m.V[: m0.nV] = m0.V
    cod_none = np.full(m.nV, 3, dtype=np.int32)
    out = {"gpu": gpu_info(), "scene": f"C5, {m.nT} tets, {args.points} codimension-0 points", "reps": args.reps}
    ctxs, gids = {}, {}
    for with_pts in (False, True):
        ctx = L.Context(0)
        ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
        ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim if with_pts else cod_none)
        ctx.set_state(m.V_soa)
        n0 = ctx.launch_count()
        ctx.intersection_free(want=False)  # eager first: lazy allocations
        out[f"launches_{'with' if with_pts else 'without'}_points"] = ctx.launch_count() - n0
        out[f"count_{'with' if with_pts else 'without'}_points"] = ctx.fetch_iteration().n_intersected_triangles
        ctx.capture_begin()
        ctx.intersection_free(want=False)
        gids[with_pts] = ctx.capture_end()
        ctxs[with_pts] = ctx
    times = {False: [], True: []}
    for _ in range(args.reps):
        for with_pts in (False, True):
            ctx = ctxs[with_pts]
            ctx.sync()
            ctx.timer_start()
            ctx.graph_launch(gids[with_pts])
            times[with_pts].append(ctx.timer_stop())
            ctx.fetch_iteration()
    out["intersection_free_without_points_ms"] = med(times[False])
    out["intersection_free_with_points_ms"] = med(times[True])
    out["point_in_tet_stage_ms"] = med(times[True]) - med(times[False])
    print(json.dumps(out))
    for with_pts, ctx in ctxs.items():
        ctx.graph_destroy(gids[with_pts])
        ctx.close()


if __name__ == "__main__":
    main()

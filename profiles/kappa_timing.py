"""Cost of the device-resident barrier stiffness on C5 (146 x sphere1K.msh, 1M tets): ipcgpu_set_kappa, ipcgpu_kappa_init (g_c, the two
fixed-order dot products and the decision; g_E left by the NULL-output elastic gradient), ipcgpu_kappa_clear_close_set and
ipcgpu_kappa_post_line_search (check, doubling, snapshot), each timed alone with device events around it on the context stream (medians
over --reps), plus the close-set size and the active-set size they ran on.  Prints one JSON line with the card's name, SM clock and power
limit read in the same run.
    python profiles/kappa_timing.py [--reps 20]"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import oracle_kappa as ok  # noqa: E402
from device_pattern_timing import Args, gpu_info, med  # noqa: E402
from ipc_b200 import lib as L  # noqa: E402

DT2 = 0.025 ** 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    m, info = bench.build_scene(Args())
    dHat = info["dHat"]
    ctx = L.Context(0)
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_canonical_order(0)
    ctx.set_state(m.V_soa)
    nC, _, _ = ctx.constraint_set(dHat, 1, fetch=False)
    ctx.elastic_gradient(DT2, 1, 1, want=False)
    s, mx = ok.bounds(dHat, 1e-11, float(np.mean(m.mass)), float(np.sum((m.V_rest.max(0) - m.V_rest.min(0)) ** 2)))

    def timed(fn):
        fn()  # warm-up (lazy allocations)
        t = []
        for _ in range(args.reps):
            ctx.timer_start()
            fn()
            t.append(ctx.timer_stop())
        return med(t)

    out = {"gpu": gpu_info(), "scene": f"C5, {m.nT} tets, {m.nV} vertices, {nC} active pairs", "reps": args.reps}
    out["set_kappa_ms"] = timed(lambda: ctx.set_kappa(s, s, mx))
    out["kappa_init_ms"] = timed(lambda: ctx.kappa_init(dHat))
    out["clear_close_set_ms"] = timed(ctx.kappa_clear_close_set)
    out["post_line_search_ms"] = timed(lambda: ctx.kappa_post_line_search(dHat))  # (dTol = dHat: every active pair is saved)
    k = ctx.kappa_info()
    out["n_close"], out["kappa"], out["doublings"] = k.n_close, k.kappa, k.doublings
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()

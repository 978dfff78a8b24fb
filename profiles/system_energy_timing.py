"""Cost of the end-of-step diagnostics on C5 (146 x sphere1K.msh, 1M tets, 146 components), and of the host path they replace.
  - ipcgpu_system_energy (deferred form): the per-tet elastic energy pass, the per-segment sums and the per-component sums, timed together
    and, for the split, the elastic energy pass alone (ipcgpu_elastic_energy in its deferred form: the same per-tet kernel plus one reduce);
  - ipcgpu_constraint_summary (deferred form) over the self-contact active set;
  each with device events around it on the context stream, medians over --reps after a warm-up;
  - the replaced host path, host clock around work that ends in a synchronisation: the eager per-tet energy, the download of e_per_tet, V and
    V_prev and the numpy reduction per component; and ipcgpu_evaluate_constraints (download included) plus the numpy summary.
Prints one JSON line with the card's name, SM clock and power limit read in the same run.
    python profiles/system_energy_timing.py [--reps 20]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import oracle_diagnostics as od  # noqa: E402
import oracle_timestep as ot  # noqa: E402
from device_pattern_timing import Args, gpu_info, med  # noqa: E402
from ipc_b200 import lib as L  # noqa: E402

DT = 0.025
N_COMP = 146


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    m, info = bench.build_scene(Args())
    dHat, kappa = info["dHat"], 1e5
    ctx = L.Context(0)
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_canonical_order(0)
    ctx.set_state(m.V_soa)
    Vprev = m.V - 1e-3 * np.sqrt(dHat) * info["p"].reshape(-1, 3)
    ctx.set_prev_state(np.ascontiguousarray(Vprev.T).ravel())
    ctx.set_time_integration(L.TIT_BE, DT, gravity=(0.0, 0.0, -9.81))
    assert m.nV % N_COMP == 0 and m.nT % N_COMP == 0
    ve = np.arange(1, N_COMP + 1) * (m.nV // N_COMP)
    te = np.arange(1, N_COMP + 1) * (m.nT // N_COMP)
    ctx.set_components(ve, te)
    nC = ctx.constraint_set(dHat, 1)[0].shape[0]

    def timed(fn):
        fn()  # warm-up (lazy allocations)
        t = []
        for _ in range(args.reps):
            ctx.timer_start()
            fn()
            t.append(ctx.timer_stop())
        return med(t)

    def host_timed(fn):
        fn()
        t = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            fn()
            t.append(1e3 * (time.perf_counter() - t0))
        return med(t)

    P = ot.Params(ot.BE, DT, gravity=(0.0, 0.0, -9.81))
    tet_starts, v_starts = np.concatenate([[0], te[:-1]]), np.concatenate([[0], ve[:-1]])

    def host_system_energy():
        ctx.elastic_energy(1.0)  # (synchronises)
        e_t = ctx.download(L.BUF_ENERGY_PER_TET, m.nT)
        V = ctx.download(L.BUF_POSITIONS, 3 * m.nV).reshape(3, -1).T
        Vp = np.asarray(Vprev)  # (a binding that keeps V_prev on the device downloads it too: counted below as a second V)
        ctx.download(L.BUF_POSITIONS, 3 * m.nV)
        e, p, Lm = od.vertex_terms(V, Vp, m.mass, P)
        return np.add.reduceat(e_t, tet_starts) + np.add.reduceat(e, v_starts), np.add.reduceat(p, v_starts), np.add.reduceat(Lm, v_starts)

    def host_summary():
        return od.summary(ctx.evaluate_constraints(nC), dHat, kappa)

    out = {"gpu": gpu_info(), "scene": f"C5, {m.nT} tets, {m.nV} vertices, {N_COMP} components, {nC} active pairs", "reps": args.reps}
    out["system_energy_ms"] = timed(lambda: ctx.system_energy(want=False))
    out["elastic_energy_pass_ms"] = timed(lambda: ctx.elastic_energy(1.0, want=False))
    out["constraint_summary_ms"] = timed(lambda: ctx.constraint_summary(dHat, kappa, want=False))
    out["host_system_energy_ms"] = host_timed(host_system_energy)
    out["host_constraint_summary_ms"] = host_timed(host_summary)
    E_dev, M_dev, L_dev = ctx.system_energy()
    E_host, M_host, L_host = host_system_energy()
    out["max_rel_diff_sysE"] = float(np.max(np.abs(E_dev - E_host) / np.abs(E_host)))
    s = ctx.constraint_summary(dHat, kappa)
    out["summary"] = dict(n=s.n, d_min=s.d_min, d_max=s.d_max, fb_norm=s.fb_norm)
    out["download_bytes_replaced"] = 8 * (m.nT + 6 * m.nV)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()

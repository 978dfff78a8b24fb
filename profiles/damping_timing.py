"""Cost of the Rayleigh-damping stages at C5 (146 x sphere1K.msh, 1M tets), device events around each call (ipcgpu_timer_start / _stop), medians:
  1. ipcgpu_damping_update (per-tet Hessian + assembly into slot storage: once per time step);
  2. per Newton iteration: the damping energy, gradient (D d) and Hessian (D added into the CSR);
  3. one eager line search with damping on and off (the same entry state; the host drives its loops, so the time includes its decisions).
The bytes of each per-iteration call are counted from the slot count (9 doubles per slot, the index words and the vertex arrays each call
reads and writes once) and divided by the measured time.  Prints one JSON line with the card's name, SM clock and power limit read in the same run.
    python profiles/damping_timing.py [--reps 20]"""
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


def timed(ctx, f, reps):
    out = []
    for _ in range(reps):
        ctx.timer_start()
        f()
        out.append(ctx.timer_stop())
    return med(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    m, info = bench.build_scene(Args())
    dHat, kappa = info["dHat"], bench.KAPPA
    ia, ja = m.csr_pattern(1)
    nV, nnz = m.nV, ja.size
    n_off = (nnz - 6 * nV) // 9  # off-diagonal vertex pairs of the mesh pattern
    n_slots = nV + n_off
    P = np.array(info["p"], dtype=np.float64).reshape(-1, 3)
    ctx = L.Context(0)
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_csr(ia, ja, 1)
    ctx.set_state(m.V_soa)
    ctx.set_prev_state(np.ascontiguousarray((m.V - 1e-2 * P).T).ravel())
    ctx.set_search_dir(np.ascontiguousarray(P).ravel())
    coef = 0.1
    ctx.damping_update(coef)  # first call: slot incidence
    res = dict(metric="damping_c5", gpu=gpu_info(), nV=nV, nT=m.nT, slots=n_slots, reps=args.reps)
    res["update_ms"] = timed(ctx, lambda: ctx.damping_update(coef), args.reps)
    res["energy_ms"] = timed(ctx, lambda: ctx.damping_energy(want=False), args.reps)
    res["gradient_ms"] = timed(ctx, lambda: ctx.damping_gradient(1), args.reps)
    res["hessian_ms"] = timed(ctx, lambda: ctx.damping_hessian(), args.reps)
    # bytes: D once (energy, Hessian) or twice for an off-diagonal block (gradient: both of its vertices gather it)
    vec = 8 * 3 * nV
    b_energy = n_slots * (72 + 8) + 2 * vec + 8 * (n_slots // 256)
    b_grad = (n_slots + n_off) * (72 + 8) + 4 * (nV + 1) + 2 * vec + 2 * vec
    b_hess = n_off * 72 + nV * 48 + n_slots * (8 + 12) + 16 * nnz
    for k, b in (("energy", b_energy), ("gradient", b_grad), ("hessian", b_hess)):
        res[k + "_bytes"] = int(b)
        res[k + "_GBps"] = round(b / (res[k + "_ms"] * 1e-3) / 1e9, 1)

    def ls():
        ctx.set_state(m.V_soa)
        ctx.constraint_set(dHat, 1, fetch=False, sizes=False)
        ctx.step_bound_set(1.0)
        ctx.timer_start()
        ctx.line_search(DT2, dHat, kappa, check=False)
        return ctx.timer_stop()

    on, off = [], []
    for _ in range(max(3, args.reps // 4)):
        ctx.damping_update(coef)
        on.append(ls())
        ctx.damping_update(0.0)
        off.append(ls())
    res["line_search_damping_on_ms"], res["line_search_damping_off_ms"] = med(on), med(off)
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()

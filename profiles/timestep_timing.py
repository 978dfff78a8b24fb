"""Cost of the time-integration frame of a time step at C5 (146 x sphere1K.msh, 1M tets), the end of a time step followed by the warm start
(initX option 1, backward Euler), three ways:
  1. device: ipcgpu_end_time_step + ipcgpu_warm_start(1), enqueued eagerly (the host drives the two loops' decisions);
  2. device, replayed: the same two calls captured once into a CUDA graph (the loops are conditional nodes);
  3. host-driven: download V, the numpy update of tests/oracle_timestep.py (dx_Elastic, velocity, acceleration, V_prev, x~, predictor), upload
     x~, V_prev and p, then the step bound and the two loops through the existing synchronous entry points.
Every repetition starts from the same state (reset outside the timed window).  Each is timed with device events on the context's stream and with
the host clock around work that ends in a synchronisation; medians and min-max.  The end-of-step kernel alone is timed as well, with the bytes it
moves (ten 3 nV double arrays).  Prints one JSON line with the card's name, SM clock and power limit read in the same run.
    python profiles/timestep_timing.py [--reps 15]"""
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
import oracle_timestep as OT  # noqa: E402
from device_pattern_timing import Args, gpu_info  # noqa: E402
from ipc_b200 import lib as L  # noqa: E402

TOL = 1e-6
DT = 0.01


def stats(x):
    return dict(median=float(np.median(x)), min=float(np.min(x)), max=float(np.max(x)))


def soa(A):
    return np.ascontiguousarray(np.asarray(A).T).ravel()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    m, info = bench.build_scene(Args())
    nV, voxel = m.nV, m.avgEdgeLen / 3.0
    P = OT.Params(OT.BE, DT, gravity=(0.0, -9.81, 0.0))
    vel0 = np.array(info["p"], dtype=np.float64).reshape(-1, 3) / DT  # the squeeze of the pile as the last step's velocity
    V0 = m.V.copy()
    # where the Newton iterations of the last step left the state: 2 % of the squeeze, so that facing balls (gaps >= 0.3 sqrt(dHat), each
    # moving <= 3 sqrt(dHat) toward the other) stay apart and the predictor (the same 2 %) is a small, contact-free motion
    V1 = V0 + 0.02 * DT * vel0
    evf, eee = L.Context.ti_error(m.V_soa, nV, None)
    ctx = L.Context(0)
    ctx.set_mesh(m.V_rest_soa, m.T_soa, m.restTriInv, m.vol, m.mu, m.lam, m.mass, m.dbc, m.energy)
    ctx.set_surface(m.SVI, m.SFEdges, m.SF_soa, m.vCoDim)
    ctx.set_time_integration(P.type, P.dt, P.beta, P.gamma, P.gravity)
    ctx.set_canonical_order(0)
    xt0 = OT.xtilde(P, V0, vel0, np.zeros_like(vel0), m.dbc)

    def reset():
        ctx.set_state(soa(V1))
        ctx.set_prev_state(soa(V0))
        ctx.set_dynamics(vel0.ravel(), None, None)
        ctx.compute_xtilde()
        ctx.sync()

    def device_frame():
        ctx.end_time_step()
        ctx.warm_start(1, voxel, TOL, evf, eee, want=False)

    def host_frame():
        V = ctx.download(L.BUF_POSITIONS, 3 * nV).reshape(3, nV).T
        vel, acc, dxe, Vp, xt = OT.end_time_step(P, V, V0, xt0, vel0, np.zeros_like(vel0), m.dbc)
        ctx.set_xtilde(soa(xt))
        ctx.set_prev_state(soa(Vp))
        ctx.set_search_dir(np.ascontiguousarray(OT.predictor(P, 1, vel, dxe, m.dbc)).ravel())
        a = ctx.inversion_step(None, 0.2, 1.0) if m.energy == 0 else 1.0
        a = ctx.hash_build_swept(None, a, voxel)
        a, _ = ctx.ccd_full(TOL, evf, eee, a)
        ctx.save_state()
        ctx.step_forward(None, a)
        while m.energy == 0 and ctx.check_inversion() > 0 and a > 0.0:  # (the reference would spin at 0; the device stops there)
            a /= 2.0
            ctx.step_forward(None, a)
        while not ctx.intersection_free() and a > 0.0:
            a /= 2.0
            ctx.step_forward(None, a)
        return a

    def timed(f, what):
        print(what, file=sys.stderr, flush=True)
        dev, host = [], []
        for _ in range(args.reps):
            reset()
            t0 = time.perf_counter()
            ctx.timer_start()
            f()
            dev.append(ctx.timer_stop())  # (synchronises)
            host.append((time.perf_counter() - t0) * 1e3)
        return dict(device_ms=stats(dev), host_ms=stats(host))

    res = dict(metric="timestep_frame_c5", gpu=gpu_info(), nV=nV, nT=m.nT, reps=args.reps)
    print("scene built, warm-up", file=sys.stderr, flush=True)
    reset()
    device_frame()  # warm-up: lazy allocations, the streams of the conditional nodes
    it = ctx.fetch_iteration()
    info_d = ctx.step_control_info()
    res["device_alpha"], res["device_status"] = info_d.alpha, info_d.status
    res["alpha_full_ccd"] = it.alpha_full_ccd
    reset()
    res["host_alpha"] = host_frame()
    ctx.fetch_iteration()
    res["eager"] = timed(device_frame, "eager")
    reset()
    ctx.capture_begin()
    device_frame()
    gid = ctx.capture_end()
    res["replayed"] = timed(lambda: ctx.graph_launch(gid), "replayed")
    res["host_driven"] = timed(host_frame, "host-driven")
    # the end-of-step kernel alone (no loop decisions): bytes of the ten 3 nV arrays it reads or writes
    res["end_time_step"] = timed(ctx.end_time_step, "end_time_step")
    nbytes = 10 * 3 * nV * 8
    res["end_time_step_bytes"] = nbytes
    res["end_time_step_TBps"] = nbytes / (res["end_time_step"]["device_ms"]["median"] * 1e-3) / 1e12
    ctx.graph_destroy(gid)
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

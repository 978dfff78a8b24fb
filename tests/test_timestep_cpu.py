"""CPU checks of the time-integration restatement (tests/oracle_timestep.py) that the GPU tests compare against, and of the C ABI of the new
calls: a free fall with V = x~ at every step (the exact minimiser of an inertia-only time step) follows the same recurrence in exact rational
arithmetic and the closed-form trajectory; the ctypes signatures of the new entry points match include/ipcgpu.h."""
import os
import re
from fractions import Fraction as Fr

import numpy as np
import pytest

import oracle_timestep as OT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = (0.3, -9.81, 0.7)
# (type, beta, gamma): the reference's defaults (Config.hpp:96) and a non-default Newmark pair
PARAMS = [(OT.BE, 0.25, 0.5), (OT.NM, 0.25, 0.5), (OT.NM, 0.3, 0.6)]


def exact_end_step(P, V, Vprev, xt, vel, acc):
    """the same recurrence over Fractions (row-wise lists of 3)"""
    dt, beta, gamma = Fr(P.dt), Fr(P.beta), Fr(P.gamma)
    g = [Fr(x) for x in P.gravity]
    dtSq = dt * dt
    if P.type == OT.BE:
        vn = [[(V[v][d] - Vprev[v][d]) / dt for d in range(3)] for v in range(len(V))]
        an = [[(vn[v][d] - vel[v][d]) / dt for d in range(3)] for v in range(len(V))]
        xtn = [[V[v][d] + (vn[v][d] * dt + dtSq * g[d]) for d in range(3)] for v in range(len(V))]
    else:
        an = [[(V[v][d] - xt[v][d]) / (dtSq * beta) + g[d] for d in range(3)] for v in range(len(V))]
        vn = [[vel[v][d] + dt * (1 - gamma) * acc[v][d] + dt * gamma * an[v][d] for d in range(3)] for v in range(len(V))]
        xtn = [[V[v][d] + (vn[v][d] * dt + beta * dtSq * g[d] + (Fr(1, 2) - beta) * dtSq * an[v][d]) for d in range(3)] for v in range(len(V))]
    return vn, an, [row[:] for row in V], xtn


@pytest.mark.parametrize("typ,beta,gamma", PARAMS)
def test_free_fall_matches_exact_arithmetic(typ, beta, gamma):
    K, dt = 40, 0.01
    P = OT.Params(typ, dt, beta, gamma, G)
    rng = np.random.default_rng(3)
    x0, v0 = rng.standard_normal((5, 3)), rng.standard_normal((5, 3))
    a0 = np.tile(P.gravity, (5, 1))  # a Newmark run starts from a = g: then x~ is the exact projectile
    # float64 oracle
    Vp, vel, acc = x0.copy(), v0.copy(), a0.copy()
    xt = OT.xtilde(P, Vp, vel, acc)
    # exact recurrence on the same (rounded) parameters
    q = OT.Params(typ, dt, beta, gamma, G)
    fx = lambda A: [[Fr(float(x)) for x in row] for row in A]
    eVp, evel, eacc = fx(x0), fx(v0), fx(a0)
    dtq, gq = Fr(q.dt), [Fr(float(x)) for x in q.gravity]
    if typ == OT.BE:
        ext = [[eVp[v][d] + (evel[v][d] * dtq + dtq * dtq * gq[d]) for d in range(3)] for v in range(5)]
    else:
        bq = Fr(q.beta)
        ext = [[eVp[v][d] + (evel[v][d] * dtq + bq * dtq * dtq * gq[d] + (Fr(1, 2) - bq) * dtq * dtq * eacc[v][d]) for d in range(3)] for v in range(5)]
    for _ in range(K):
        V = xt.copy()  # argmin of the inertia term alone
        vel, acc, dxe, Vp, xt = OT.end_time_step(P, V, Vp, xt, vel, acc)
        assert not dxe.any()
        eV = [row[:] for row in ext]
        evel, eacc, eVp, ext = exact_end_step(q, eV, eVp, ext, evel, eacc)
    exact = np.array([[float(x) for x in row] for row in eVp])
    scale = np.abs(x0).max() + K * dt * np.abs(v0).max() + (K * dt) ** 2 * 10.0
    np.testing.assert_allclose(Vp, exact, rtol=0, atol=64 * K * np.finfo(float).eps * scale)
    # ... and the exact recurrence is the closed-form trajectory: BE x_K = x0 + K dt v0 + dt^2 g K(K+1)/2, Newmark from a = g: + dt^2 g K^2/2
    c = Fr(K * (K + 1), 2) if typ == OT.BE else Fr(K * K, 2)
    closed = [[Fr(float(x0[v, d])) + K * dtq * Fr(float(v0[v, d])) + dtq * dtq * gq[d] * c for d in range(3)] for v in range(5)]
    assert eVp == closed


def test_dirichlet_vertices_and_option_zero():
    P = OT.Params(OT.NM, 0.02, 0.3, 0.6, G)
    rng = np.random.default_rng(1)
    Vp, vel, acc, dxe = (rng.standard_normal((6, 3)) for _ in range(4))
    dbc = np.array([0, 1, 2, 0, 1, 0], np.uint8)
    xt = OT.xtilde(P, Vp, vel, acc, dbc)
    assert np.array_equal(xt[dbc != 0], Vp[dbc != 0]) and not np.array_equal(xt[dbc == 0], Vp[dbc == 0])
    for option in range(5):
        p = OT.predictor(P, option, vel, dxe, dbc)
        assert not p[dbc != 0].any()
        assert p[dbc == 0].any() == (option > 0)
    with pytest.raises(ValueError):
        OT.predictor(P, 5, vel, dxe, dbc)


def header_prototypes():
    src = open(os.path.join(ROOT, "include", "ipcgpu.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return {m.group(1): [a.strip() for a in m.group(2).split(",")] for m in re.finditer(r"\bint\s+(ipcgpu_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src)}


NEW = ["ipcgpu_set_time_integration", "ipcgpu_set_dynamics", "ipcgpu_get_dynamics", "ipcgpu_compute_xtilde", "ipcgpu_end_time_step", "ipcgpu_warm_start"]


def test_new_signatures_match_the_header():
    import ctypes as C
    from ipc_b200 import lib as L
    protos = header_prototypes()
    for name in NEW:
        args = protos[name]
        res, argtypes = L.SIGNATURES[name]
        assert res is C.c_int and len(argtypes) == len(args), name
        for a, t in zip(args, argtypes):
            if "ipcgpu_ctx*" in a:
                assert t is C.c_void_p
            elif "*" in a or "[3]" in a:
                assert t is C.POINTER(C.c_double), (name, a)
            elif a.startswith("double"):
                assert t is C.c_double, (name, a)
            else:
                assert a.startswith("int") and t is C.c_int, (name, a)
    src = open(os.path.join(ROOT, "include", "ipcgpu.h")).read()
    for k, v in (("IPCGPU_BUF_POSITIONS", L.BUF_POSITIONS), ("IPCGPU_BUF_SEARCH_DIR", L.BUF_SEARCH_DIR), ("IPCGPU_BUF_XTILDE", L.BUF_XTILDE)):
        assert re.search(rf"\b{k}\s*=\s*{v}\b", src), k


def test_new_symbols_exported():
    from ipc_b200 import lib as L
    lib = L.load()
    for name in NEW:
        assert hasattr(lib, name), name

"""Float64 restatement of the end-of-step diagnostics (the oracle of csrc/diagnostics.cu). TEST INFRASTRUCTURE ONLY.

  - Optimizer::computeSystemEnergy (Optimizer.cpp:3746-3778): per vertex, m (|V - V_prev|^2 / dtSq / 2 - g.V), p = m / dt (V - V_prev) and
    V x p, each in the evaluation order of the reference's Eigen expressions (numpy rounds every elementwise operation once, no fused
    multiply-add): the squared norm adds the squares left to right, the fixed-size dot is the unrolled redux g0 x0 + (g1 x1 + g2 x2);
    per component the sums over its tets and vertices with math.fsum (the correctly rounded sum, which the device's fixed-order sum is
    measured against) and the sum of the absolute terms (the scale of its rounding);
  - the Fischer-Burmeister residual of the read-back after solveSub_IP (:1681-1692): fb = dual + d - sqrt(dual^2 + d^2) with
    dual = -kappa g_b(d, dHat) and g_b = g_bC2 (BarrierFunctions.hpp:61-71).
Positions are (nV, 3) arrays; Params is oracle_timestep.Params (dt, dtSq = dt * dt, gravity).
"""
import math

import numpy as np


def vertex_terms(V, Vprev, mass, P):
    """-> (e (nV,), p (nV, 3), L (nV, 3)): the per-vertex terms of computeSystemEnergy"""
    V = np.asarray(V, dtype=np.float64)
    dx = V - np.asarray(Vprev, dtype=np.float64)
    mass = np.asarray(mass, dtype=np.float64)
    g = P.gravity
    sq = (dx[:, 0] * dx[:, 0] + dx[:, 1] * dx[:, 1]) + dx[:, 2] * dx[:, 2]
    gx = g[0] * V[:, 0] + (g[1] * V[:, 1] + g[2] * V[:, 2])
    e = mass * (sq / P.dtSq / 2.0 - gx)
    p = (mass / P.dt)[:, None] * dx
    L = np.stack([V[:, 1] * p[:, 2] - V[:, 2] * p[:, 1], V[:, 2] * p[:, 0] - V[:, 0] * p[:, 2], V[:, 0] * p[:, 1] - V[:, 1] * p[:, 0]], axis=1)
    return e, p, L


def ranges(ends):
    lo = 0
    for hi in ends:
        yield lo, int(hi)
        lo = int(hi)


def system_energy(e_per_tet, V, Vprev, mass, P, vertex_end, tet_end):
    """-> dict of per-component arrays: E_el, E_v (sysE = E_el + E_v), M (n, 3), L (n, 3), each with its absolute-term scale (*_abs)"""
    e, p, L = vertex_terms(V, Vprev, mass, P)
    e_t = np.asarray(e_per_tet, dtype=np.float64)
    n = len(vertex_end)
    out = {k: np.zeros(n) for k in ("E_el", "E_el_abs", "E_v", "E_v_abs")}
    out.update({k: np.zeros((n, 3)) for k in ("M", "M_abs", "L", "L_abs")})
    for c, ((tl, th), (vl, vh)) in enumerate(zip(ranges(tet_end), ranges(vertex_end))):
        out["E_el"][c] = math.fsum(e_t[tl:th])
        out["E_el_abs"][c] = math.fsum(np.abs(e_t[tl:th]))
        out["E_v"][c] = math.fsum(e[vl:vh])
        out["E_v_abs"][c] = math.fsum(np.abs(e[vl:vh]))
        for d in range(3):
            out["M"][c, d] = math.fsum(p[vl:vh, d])
            out["M_abs"][c, d] = math.fsum(np.abs(p[vl:vh, d]))
            out["L"][c, d] = math.fsum(L[vl:vh, d])
            out["L_abs"][c, d] = math.fsum(np.abs(L[vl:vh, d]))
    return out


def g_b(d, dHat):
    """g_bC2 (BarrierFunctions.hpp:61-71)"""
    t2 = d - dHat
    return t2 * np.log(d / dHat) * -2.0 - (t2 * t2) / d


def fb(d, dHat, kappa):
    """the Fischer-Burmeister residual per constraint value (:1684-1691) -> (fb, |dual| + d, the scale of its cancellation)"""
    d = np.asarray(d, dtype=np.float64)
    dual = g_b(d, dHat) * -kappa
    return dual + d - np.sqrt(dual * dual + d * d), np.abs(dual) + d


def summary(d, dHat, kappa):
    """(n, d_min, d_max, |fb|, the scale |(|dual| + d)|) over the constraint values d; zeros for none"""
    d = np.asarray(d, dtype=np.float64)
    if d.size == 0:
        return 0, 0.0, 0.0, 0.0, 0.0
    f, s = fb(d, dHat, kappa)
    return int(d.size), float(d.min()), float(d.max()), math.sqrt(math.fsum(f * f)), math.sqrt(math.fsum(s * s))


def plane_d2(par, V, act):
    """the squared distance of every (plane, vertex) entry as the half-space kernels evaluate it"""
    act = np.asarray(act, dtype=np.int64).reshape(-1, 2)
    pl, x = par[act[:, 0]], np.asarray(V)[act[:, 1]]
    dist = ((pl[:, 0] * x[:, 0] + pl[:, 1] * x[:, 1]) + pl[:, 2] * x[:, 2]) + pl[:, 3]
    return dist * dist

"""float64 restatement of the reference's adaptive barrier stiffness (ADAPTIVE_KAPPA): suggestKappa / upperBoundKappa (Optimizer.cpp:2216-2233),
initKappa (:2236-2313) and postLineSearch (:2357-2445).  Distances and Jacobians come from the CPU oracle (oracle.py); the plane distances are
evaluated as HalfSpace does, one rounding per operation.  TEST INFRASTRUCTURE ONLY."""
import math

import numpy as np

import oracle as orc


def H_b(d, dHat):
    """H_bC2 (BarrierFunctions.hpp:73-83)"""
    t2 = d - dHat
    return (math.log(d / dHat) * -2.0 - t2 * 4.0 / d) + 1.0 / (d * d) * (t2 * t2)


def bounds(dHat, kappa_min_multiplier, avg_node_mass, bbox_diag2):
    """(suggestKappa, kappaMax of upperBoundKappa), in the reference's left-to-right order"""
    Hb = H_b(1.0e-16 * bbox_diag2, dHat)
    return (kappa_min_multiplier * avg_node_mass / (4.0e-16 * bbox_diag2 * Hb),
            100 * kappa_min_multiplier * avg_node_mass / (4.0e-16 * bbox_diag2 * Hb))


def stencil(mm):
    """MMCVID -> (kind, vertex ids, multiplicity)"""
    x, y, z, w = (int(v) for v in mm)
    if x >= 0:
        return "EE", [x, y, z, w], 1.0
    v0 = -x - 1
    if z < 0:
        return "PP", [v0, y], float(-w)
    if w < 0:
        return "PE", [v0, y, z], float(-w)
    return "PT", [v0, y, z, w], 1.0


def pair_d2(V, mm):
    kind, vs, _ = stencil(mm)
    return orc.d_pair(kind, V[vs])


def plane_d2(par, V, e):
    pl, x = par[int(e[0])], V[int(e[1])]
    dist = ((pl[0] * x[0] + pl[1] * x[1]) + pl[2] * x[2]) + pl[3]
    return dist * dist


def constraint_gradient(V, dbc, mm, dHat, par=None, act=()):
    """g_c of initKappa: J^T g_b(d) over the self / obstacle active set and the planes' active set, the rows of every Dirichlet vertex zeroed"""
    gc = np.zeros_like(V)
    for e in mm:
        kind, vs, mult = stencil(e)
        X = V[vs]
        db = orc.barrier(orc.d_pair(kind, X), dHat)[1]
        gc[vs] += (mult * db) * orc.g_pair(kind, X).reshape(-1, 3)
    for e in act:
        pl, v = par[int(e[0])], int(e[1])
        x = V[v]
        dist = ((pl[0] * x[0] + pl[1] * x[1]) + pl[2] * x[2]) + pl[3]
        db = orc.barrier(dist * dist, dHat)[1]
        gc[v] += (db * 2.0 * dist) * pl[:3]
    gc[np.asarray(dbc) != 0] = 0.0
    return gc.ravel()


def init(kappa, suggest, kmax, gE, gc, n_active):
    """initKappa: (kappa, minKappa or None when nothing is active)"""
    if n_active == 0:
        return kappa, None
    with np.errstate(divide="ignore", invalid="ignore"):
        minK = float(-np.float64(np.dot(gc, gE)) / np.float64(np.dot(gc, gc)))
    if minK > 0.0:
        kappa = minK
    if kappa < suggest:
        kappa = suggest
    if kappa > kmax:
        kappa = kmax
    return kappa, minK


class CloseSet:
    """postLineSearch's state: kappa, its cap and the saved close entries (('mm', MMCVID) or ('hs', (plane, vertex)), d)"""

    def __init__(self, kappa, kmax):
        self.kappa, self.kmax, self.saved, self.doublings, self.needs_init = kappa, kmax, [], 0, False

    def d2(self, V, par, key):
        return pair_d2(V, key[1]) if key[0] == "mm" else plane_d2(par, V, key[1])

    def post_line_search(self, V, mm, act, dTol, par=None):
        if self.kappa == 0.0:
            self.needs_init = True
            return
        if any(self.d2(V, par, key) <= d for key, d in self.saved):
            self.kappa = min(self.kappa * 2.0, self.kmax)
            self.doublings += 1
        keys = [("mm", tuple(int(v) for v in e)) for e in mm] + [("hs", tuple(int(v) for v in e)) for e in act]
        self.saved = [(k, d) for k, d in ((k, self.d2(V, par, k)) for k in keys) if d < dTol]

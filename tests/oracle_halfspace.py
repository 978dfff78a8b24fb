"""ctypes wrapper of the half-space part of the CPU oracle (oracle/halfspace.cpp). TEST INFRASTRUCTURE ONLY."""
import ctypes as C

import numpy as np

import oracle as orc
from oracle import d, i


def planes(origin, normal, velocitydt=None, friction=None):
    """HalfSpace::init of every plane -> (n, 8) parameters [n0 n1 n2 D v0 v1 v2 mu]"""
    origin, normal = (np.ascontiguousarray(np.asarray(x, dtype=np.float64).reshape(-1, 3)) for x in (origin, normal))
    n = len(origin)
    vdt = None if velocitydt is None else np.ascontiguousarray(np.asarray(velocitydt, dtype=np.float64).reshape(-1, 3))
    fr = np.ascontiguousarray(np.zeros(n) if friction is None else np.asarray(friction, dtype=np.float64))
    par = np.zeros((n, 8))
    orc.lib().orc_hs_planes(n, d(origin), d(normal), d(vdt) if vdt is not None else None, d(fr), d(par))
    return par


class HalfSpaces:
    """the oracle's restatement over an oracle.Surf (positions, Dirichlet flags, SVI, codimensions)"""

    def __init__(self, surf, par):
        self.surf, self.par = surf, np.ascontiguousarray(par, dtype=np.float64)
        self.nP = len(self.par)

    def constraint_set(self, dHat):
        act = np.empty((max(self.nP * self.surf.SVI.size, 1), 2), dtype=np.int32)
        n = orc.lib().orc_hs_constraint_set(C.byref(self.surf.s), self.nP, d(self.par), C.c_double(dHat), i(act))
        return act[:n].copy()

    def energy(self, act, dHat, kappa):
        E = C.c_double()
        bad = orc.lib().orc_hs_energy(C.byref(self.surf.s), d(self.par), i(np.ascontiguousarray(act, dtype=np.int32)), len(act), C.c_double(dHat),
                                      C.c_double(kappa), C.byref(E))
        return E.value, bad

    def gradient(self, act, dHat, kappa, g=None):
        g = np.zeros(3 * self.surf.mesh.nV) if g is None else g
        orc.lib().orc_hs_gradient(C.byref(self.surf.s), d(self.par), i(np.ascontiguousarray(act, dtype=np.int32)), len(act), C.c_double(dHat), C.c_double(kappa), d(g))
        return g

    def hessian_csr(self, act, dHat, kappa, ia, ja, base, projectDBC=1, a=None):
        ia, ja = (np.ascontiguousarray(x, dtype=np.int32) for x in (ia, ja))
        a = np.zeros(ja.size) if a is None else a
        orc.lib().orc_hs_hessian_csr(C.byref(self.surf.s), d(self.par), i(np.ascontiguousarray(act, dtype=np.int32)), len(act), C.c_double(dHat), C.c_double(kappa),
                                     projectDBC, i(ia), i(ja), base, d(a))
        return a

    def step(self, p, slackness, alpha):
        a = C.c_double(alpha)
        orc.lib().orc_hs_step(C.byref(self.surf.s), self.nP, d(self.par), d(np.ascontiguousarray(p, dtype=np.float64)), C.c_double(slackness), C.byref(a))
        return a.value

    def crossings(self):
        return int(orc.lib().orc_hs_crossings(C.byref(self.surf.s), self.nP, d(self.par)))

    def lag(self, act, dHat, kappa):
        act = np.ascontiguousarray(act, dtype=np.int32)
        lag, lam = np.empty((max(len(act), 1), 2), dtype=np.int32), np.empty(max(len(act), 1))
        n = orc.lib().orc_hs_lag(C.byref(self.surf.s), d(self.par), i(act), len(act), C.c_double(dHat), C.c_double(kappa), i(lag), d(lam))
        return lag[:n].copy(), lam[:n].copy()

    def friction_energy(self, Vt_soa, lag, lam, eps2):
        E = C.c_double()
        orc.lib().orc_hs_friction_energy(C.byref(self.surf.s), d(np.ascontiguousarray(Vt_soa, dtype=np.float64)), d(self.par), i(np.ascontiguousarray(lag, dtype=np.int32)),
                                         d(np.ascontiguousarray(lam)), len(lag), C.c_double(eps2), C.byref(E))
        return E.value

    def friction_gradient(self, Vt_soa, lag, lam, eps2, g=None):
        g = np.zeros(3 * self.surf.mesh.nV) if g is None else g
        orc.lib().orc_hs_friction_gradient(C.byref(self.surf.s), d(np.ascontiguousarray(Vt_soa, dtype=np.float64)), d(self.par),
                                           i(np.ascontiguousarray(lag, dtype=np.int32)), d(np.ascontiguousarray(lam)), len(lag), C.c_double(eps2), d(g))
        return g

    def friction_hessian_csr(self, Vt_soa, lag, lam, eps2, ia, ja, base, projectDBC=1, a=None):
        ia, ja = (np.ascontiguousarray(x, dtype=np.int32) for x in (ia, ja))
        a = np.zeros(ja.size) if a is None else a
        orc.lib().orc_hs_friction_hessian_csr(C.byref(self.surf.s), d(np.ascontiguousarray(Vt_soa, dtype=np.float64)), d(self.par),
                                              i(np.ascontiguousarray(lag, dtype=np.int32)), d(np.ascontiguousarray(lam)), len(lag), C.c_double(eps2), projectDBC,
                                              i(ia), i(ja), base, d(a))
        return a


def barrier_block(pl, dist, dHat, kappa, project=1):
    H = np.empty(9)
    orc.lib().orc_hs_barrier_block(d(np.ascontiguousarray(pl, dtype=np.float64)), C.c_double(dist), C.c_double(dHat), C.c_double(kappa), project, d(H))
    return H.reshape(3, 3)


def friction_block(pl, x, xt, lam, eps2, project=1):
    H = np.empty(9)
    orc.lib().orc_hs_friction_block(d(np.ascontiguousarray(pl, dtype=np.float64)), d(np.ascontiguousarray(x, dtype=np.float64)),
                                    d(np.ascontiguousarray(xt, dtype=np.float64)), C.c_double(lam), C.c_double(eps2), project, d(H))
    return H.reshape(3, 3)


def trial_energy(hs, Vt_soa, act, dHat, kappa, lagged, eps2, E_el_in, E_b, E_f):
    """Optimizer::computeEnergyVal with planes (oracle/halfspace.cpp: orc_hs_trial_energy): ((E_el_in) + (E_b + E_plane_b)) + E_plane_f + E_f;
    lagged = (lag, lam) of the planes or None (no plane friction).  Returns (E, bad)"""
    E = C.c_double()
    act = np.ascontiguousarray(act, dtype=np.int32)
    lag, lam = lagged if lagged is not None else (np.zeros((0, 2), np.int32), np.zeros(0))
    lag = np.ascontiguousarray(lag, dtype=np.int32)
    lam = np.ascontiguousarray(lam, dtype=np.float64)
    bad = orc.lib().orc_hs_trial_energy(C.byref(hs.surf.s), d(np.ascontiguousarray(Vt_soa, dtype=np.float64)) if Vt_soa is not None else None, d(hs.par),
                                        i(act), len(act), C.c_double(dHat), C.c_double(kappa), int(lagged is not None), i(lag), d(lam), len(lag),
                                        C.c_double(eps2), C.c_double(E_el_in), C.c_double(E_b), C.c_double(E_f), C.byref(E))
    return E.value, bad

"""ctypes wrapper of the CPU oracle (oracle/liboracle.so). TEST INFRASTRUCTURE ONLY -- never imported by
the product package (ipc_b200/)."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
LIB = os.path.join(ORACLE_DIR, "liboracle.so")

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_u8p = C.POINTER(C.c_uint8)


def build():
    srcs = [os.path.join(ORACLE_DIR, f) for f in os.listdir(ORACLE_DIR) if f.endswith((".cpp", ".h"))]
    if os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(s) for s in srcs):
        return
    subprocess.check_call(["make", "-C", ORACLE_DIR, "-s"])


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(LIB)
    return _lib


class OrcMesh(C.Structure):
    _fields_ = [("nV", C.c_int), ("nT", C.c_int), ("V", _dp), ("T", _ip), ("Ainv", _dp), ("vol", _dp),
                ("mu", _dp), ("lam", _dp), ("dbc", _u8p), ("energy_type", C.c_int)]


def d(a):
    return a.ctypes.data_as(_dp)


def i(a):
    return a.ctypes.data_as(_ip)


class Elastic:
    """Keeps numpy buffers alive next to the C struct."""

    def __init__(self, mesh, V=None, energy=None, dbc=None):
        self.nV, self.nT = mesh.nV, mesh.nT
        self.V = np.ascontiguousarray((mesh.V if V is None else V).T).ravel().astype(np.float64)
        self.T = np.ascontiguousarray(mesh.T.T).ravel().astype(np.int32)
        self.A = np.ascontiguousarray(mesh.restTriInv, dtype=np.float64).ravel()
        self.vol, self.mu, self.lam = (np.ascontiguousarray(x, dtype=np.float64) for x in (mesh.vol, mesh.mu, mesh.lam))
        self.dbc = np.ascontiguousarray(mesh.dbc if dbc is None else dbc, dtype=np.uint8)
        et = mesh.energy if energy is None else energy
        self.m = OrcMesh(self.nV, self.nT, d(self.V), i(self.T), d(self.A), d(self.vol), d(self.mu), d(self.lam),
                         self.dbc.ctypes.data_as(_u8p), et)

    def energy(self, coef, nthreads=1):
        E = C.c_double()
        per = np.empty(self.nT)
        lib().orc_elastic_energy(C.byref(self.m), C.c_double(coef), d(per), C.byref(E), nthreads)
        return E.value, per

    def gradient(self, coef, projectDBC=1, nthreads=1):
        g = np.empty(3 * self.nV)
        lib().orc_elastic_gradient(C.byref(self.m), C.c_double(coef), projectDBC, d(g), nthreads)
        return g

    def count_inverted(self):
        return int(lib().orc_count_inverted(C.byref(self.m)))

    def hessian_blocks(self, coef, projectSPD=1, nthreads=1):
        H = np.empty((self.nT, 12, 12))
        lib().orc_elastic_hessian_blocks(C.byref(self.m), C.c_double(coef), projectSPD, d(H), nthreads)
        return H

    def hessian_csr(self, coef, ia, ja, base, projectSPD=1, projectDBC=1, a=None, nthreads=1):
        ia = np.ascontiguousarray(ia, dtype=np.int32)
        ja = np.ascontiguousarray(ja, dtype=np.int32)
        if a is None:
            a = np.zeros(ja.size)
        lib().orc_elastic_hessian_csr(C.byref(self.m), C.c_double(coef), projectSPD, projectDBC, i(ia), i(ja), base, d(a), nthreads)
        return a

    def inversion_step(self, p, slack, alpha):
        p = np.ascontiguousarray(p, dtype=np.float64)
        per = np.empty(self.nT)
        a = C.c_double(alpha)
        lib().orc_inversion_step(C.byref(self.m), d(p), C.c_double(slack), d(per), C.byref(a))
        return a.value, per


def svd3(F):
    F = np.ascontiguousarray(F, dtype=np.float64).ravel()
    U, S, V = np.empty(9), np.empty(3), np.empty(9)
    lib().orc_svd3(d(F), d(U), d(S), d(V))
    return U.reshape(3, 3), S, V.reshape(3, 3)


SVD3_EXITS = ("beta_2", "beta_1", "alpha_2", "alpha_3", "alpha_1")


def svd3_branch(F):
    """(exit, sort, reordered) of the restated SVD on F: the exit's name (SVD3_EXITS, in the order the exits are tested), which sort ran
    (0 after process(0), 1 after process(1)) and whether that sort took its swapping branch instead of the early return"""
    F = np.ascontiguousarray(F, dtype=np.float64).ravel()
    ex, so, re = C.c_int(), C.c_int(), C.c_int()
    lib().orc_svd3_branch(d(F), C.byref(ex), C.byref(so), C.byref(re))
    return SVD3_EXITS[ex.value], so.value, bool(re.value)


CUBIC_EXITS = ("linear", "quad_first", "quad_second", "quad_none", "cardano_real", "cardano_complex")


def cubic_branch(a, b, c, d, tol=1e-6):
    """(t, exit, fallback, passed, kept) of the restated getSmallestPositiveRealCubicRoot on the given coefficients: the root (negative
    for none), the exit's name (CUBIC_EXITS), whether the |C| == 0 fallback ran, the mask of Cardano roots with |Im t| < tol and Re t > 0,
    and the root kept (1..3, 0 for none)"""
    t, fb, ps, kp = C.c_double(), C.c_int(), C.c_int(), C.c_int()
    f = lib().orc_cubic_branch
    f.argtypes = [C.c_double] * 5 + [_dp, _ip, _ip, _ip]
    ex = f(a, b, c, d, tol, C.byref(t), C.byref(fb), C.byref(ps), C.byref(kp))
    return t.value, CUBIC_EXITS[ex], bool(fb.value), ps.value, kp.value


def psi(et, S, mu, lam):
    S = np.ascontiguousarray(S, dtype=np.float64)
    E = C.c_double()
    lib().orc_psi(et, d(S), C.c_double(mu), C.c_double(lam), C.byref(E))
    return E.value


def dpsi(et, S, mu, lam):
    S = np.ascontiguousarray(S, dtype=np.float64)
    out = np.empty(3)
    lib().orc_dpsi(et, d(S), C.c_double(mu), C.c_double(lam), d(out))
    return out


def d2psi(et, S, mu, lam):
    S = np.ascontiguousarray(S, dtype=np.float64)
    out = np.empty(9)
    lib().orc_d2psi(et, d(S), C.c_double(mu), C.c_double(lam), d(out))
    return out.reshape(3, 3)


def pk1(et, F, mu, lam):
    U, S, V = svd3(F)
    P = np.empty(9)
    lib().orc_pk1(et, d(np.ascontiguousarray(F).ravel()), d(U.ravel().copy()), d(S), d(V.ravel().copy()), C.c_double(mu), C.c_double(lam), d(P))
    return P.reshape(3, 3)


def dPdF(et, F, mu, lam, w=1.0, projectSPD=0):
    U, S, V = svd3(F)
    out = np.empty(81)
    lib().orc_dPdF(et, d(U.ravel().copy()), d(S), d(V.ravel().copy()), C.c_double(mu), C.c_double(lam), C.c_double(w), projectSPD, d(out))
    return out.reshape(9, 9)


def makePD(M):
    M = np.ascontiguousarray(M, dtype=np.float64).copy()
    lib().orc_makePD(M.shape[0], d(M))
    return M


def blocks78_to_dense(h78, tet):
    """Rebuild the dense symmetric 12x12 from the kernel's 78-scalar block layout (DESIGN.md)."""
    H = np.zeros((12, 12))
    k = 0
    for a in range(4):
        for i_ in range(3):
            for r in range(i_, 3):
                H[3 * a + i_, 3 * a + r] = H[3 * a + r, 3 * a + i_] = h78[k]
                k += 1
    for a in range(4):
        for b in range(a + 1, 4):
            blk = h78[k:k + 9].reshape(3, 3)
            k += 9
            if tet[a] > tet[b]:
                blk = blk.T
            H[3 * a:3 * a + 3, 3 * b:3 * b + 3] = blk
            H[3 * b:3 * b + 3, 3 * a:3 * a + 3] = blk.T
    return H


# ---- contact pair math -------------------------------------------------------------------------------------------
def _vec(name, v, n):
    v = np.ascontiguousarray(v, dtype=np.float64).ravel()
    out = np.empty(n)
    getattr(lib(), name)(d(v), d(out))
    return out


def d_pair(kind, v):
    return float(_vec("orc_d_" + kind, v, 1)[0])


def g_pair(kind, v):
    return _vec("orc_g_" + kind, v, {"PP": 6, "PE": 9, "PT": 12, "EE": 12}[kind])


def H_pair(kind, v):
    n = {"PP": 6, "PE": 9, "PT": 12, "EE": 12}[kind]
    return _vec("orc_H_" + kind, v, n * n).reshape(n, n)


def dType_PT(v):
    return lib().orc_dType_PT(d(np.ascontiguousarray(v, dtype=np.float64).ravel()))


def dType_EE(v):
    return lib().orc_dType_EE(d(np.ascontiguousarray(v, dtype=np.float64).ravel()))


def point_tri_d(v):
    return float(_vec("orc_point_tri_d", v, 1)[0])


def edge_edge_d(v):
    return float(_vec("orc_edge_edge_d", v, 1)[0])


def barrier(dist, dHat):
    b, g, H = C.c_double(), C.c_double(), C.c_double()
    lib().orc_barrier(C.c_double(dist), C.c_double(dHat), C.byref(b), C.byref(g), C.byref(H))
    return b.value, g.value, H.value


def ee_cross(v):
    v = np.ascontiguousarray(v, dtype=np.float64).ravel()
    c = C.c_double()
    g, H = np.empty(12), np.empty(144)
    lib().orc_ee_cross(d(v), C.byref(c), d(g), d(H))
    return c.value, g, H.reshape(12, 12)


def mollifier(v, eps_x):
    v = np.ascontiguousarray(v, dtype=np.float64).ravel()
    e = C.c_double()
    g, H = np.empty(12), np.empty(144)
    lib().orc_mollifier(d(v), C.c_double(eps_x), C.byref(e), d(g), d(H))
    return e.value, g, H.reshape(12, 12)


class OrcSurf(C.Structure):
    _fields_ = [("nV", C.c_int), ("V", _dp), ("Vrest", _dp), ("dbc", _u8p), ("nSV", C.c_int), ("SVI", _ip), ("nSE", C.c_int), ("SE", _ip),
                ("nSF", C.c_int), ("SF", _ip), ("vCoDim", _ip)]


class Surf:
    def __init__(self, mesh, V=None):
        self.mesh = mesh
        self.V = np.ascontiguousarray((mesh.V if V is None else V).T).ravel().astype(np.float64)
        self.Vr = np.ascontiguousarray(mesh.V_rest.T).ravel().astype(np.float64)
        self.dbc = np.ascontiguousarray(mesh.dbc, dtype=np.uint8)
        self.SVI = np.ascontiguousarray(mesh.SVI, dtype=np.int32)
        self.SE = np.ascontiguousarray(mesh.SFEdges, dtype=np.int32).ravel()
        self.SF = np.ascontiguousarray(mesh.SF.T, dtype=np.int32).ravel()
        self.cod = np.ascontiguousarray(mesh.vCoDim, dtype=np.int32)
        self.s = OrcSurf(mesh.nV, d(self.V), d(self.Vr), self.dbc.ctypes.data_as(_u8p), self.SVI.size, i(self.SVI), self.SE.size // 2, i(self.SE),
                         self.SF.size // 3, i(self.SF), i(self.cod))

    def constraint_set(self, dHat, nthreads=1, cap=1 << 20):
        mm = np.empty((cap, 4), dtype=np.int32); pa = np.empty((cap, 4), dtype=np.int32); pe = np.empty((cap, 2), dtype=np.int32)
        cand = np.empty((4 * cap, 2), dtype=np.int32)
        nC, nP, nK = C.c_int(), C.c_int(), C.c_int()
        rc = lib().orc_constraint_set(C.byref(self.s), C.c_double(dHat), cap, i(mm), C.byref(nC), cap, i(pa), i(pe), C.byref(nP),
                                      4 * cap, i(cand), C.byref(nK), nthreads)
        assert rc == 0, "oracle constraint-set capacity exceeded"
        return mm[:nC.value].copy(), pa[:nP.value].copy(), pe[:nP.value].copy(), cand[:nK.value].copy()

    def intersection_free(self, cell=None, nthreads=1, flags=False):
        """checkEdgeTriIntersectionIfAny: (ok, number of intersected surface triangles[, per-triangle flags])"""
        hits = C.c_int()
        fl = np.zeros(self.SF.size // 3, dtype=np.int32) if flags else None
        ok = lib().orc_intersection_free(C.byref(self.s), C.c_double(cell if cell else self.mesh.avgEdgeLen), C.byref(hits), i(fl) if flags else None, nthreads)
        return (bool(ok), hits.value, fl) if flags else (bool(ok), hits.value)

    def constraint_set_hashed(self, dHat, voxel_size, nthreads=1, cap=1 << 20):
        mm = np.empty((cap, 4), dtype=np.int32); pa = np.empty((cap, 4), dtype=np.int32); pe = np.empty((cap, 2), dtype=np.int32)
        cand = np.empty((4 * cap, 2), dtype=np.int32)
        nC, nP, nK = C.c_int(), C.c_int(), C.c_int()
        rc = lib().orc_constraint_set_hashed(C.byref(self.s), C.c_double(dHat), C.c_double(voxel_size), cap, i(mm), C.byref(nC), cap, i(pa), i(pe), C.byref(nP),
                                             4 * cap, i(cand), C.byref(nK), nthreads)
        assert rc == 0
        return mm[:nC.value].copy(), pa[:nP.value].copy(), pe[:nP.value].copy(), cand[:nK.value].copy()

    def barrier_energy(self, mm, pa, pe, dHat, kappa):
        E = C.c_double()
        mm, pa, pe = (np.ascontiguousarray(x, dtype=np.int32) for x in (mm, pa, pe))
        bad = lib().orc_barrier_energy(C.byref(self.s), i(mm), len(mm), i(pa), i(pe), len(pa), C.c_double(dHat), C.c_double(kappa), C.byref(E))
        return E.value, bad

    def barrier_gradient(self, mm, pa, pe, dHat, kappa, g=None):
        if g is None:
            g = np.zeros(3 * self.mesh.nV)
        mm, pa, pe = (np.ascontiguousarray(x, dtype=np.int32) for x in (mm, pa, pe))
        lib().orc_barrier_gradient(C.byref(self.s), i(mm), len(mm), i(pa), i(pe), len(pa), C.c_double(dHat), C.c_double(kappa), 1, d(g))
        return g

    def barrier_hessian_csr(self, mm, pa, pe, dHat, kappa, ia, ja, base, projectDBC=1, a=None, nthreads=1):
        ia = np.ascontiguousarray(ia, dtype=np.int32); ja = np.ascontiguousarray(ja, dtype=np.int32)
        if a is None:
            a = np.zeros(ja.size)
        mm, pa, pe = (np.ascontiguousarray(x, dtype=np.int32) for x in (mm, pa, pe))
        lib().orc_barrier_hessian_csr(C.byref(self.s), i(mm), len(mm), i(pa), i(pe), len(pa), C.c_double(dHat), C.c_double(kappa), projectDBC,
                                      i(ia), i(ja), base, d(a), nthreads)
        return a

    # ---- lagged friction (oracle/friction.cpp) ----
    def friction_lag(self, mm, dHat, kappa):
        """(lambda, coord (n,2), basis (n,6)) of the active set at the current positions"""
        mm = np.ascontiguousarray(mm, dtype=np.int32)
        n = len(mm)
        lam, co, ba = np.empty(max(n, 1)), np.empty((max(n, 1), 2)), np.empty((max(n, 1), 6))
        lib().orc_friction_lag(C.byref(self.s), i(mm), n, C.c_double(dHat), C.c_double(kappa), d(lam), d(co), d(ba))
        return lam[:n], co[:n], ba[:n]

    @staticmethod
    def _soa(Vt):
        return np.ascontiguousarray(np.asarray(Vt, dtype=np.float64).T).ravel() if np.ndim(Vt) == 2 else np.ascontiguousarray(Vt, dtype=np.float64)

    def friction_energy(self, Vt, mm, lam, co, ba, eps2, coef):
        mm = np.ascontiguousarray(mm, dtype=np.int32); vt = self._soa(Vt)
        lam, co, ba = (np.ascontiguousarray(x, dtype=np.float64) for x in (lam, co, ba))
        E = C.c_double()
        lib().orc_friction_energy(C.byref(self.s), d(vt), i(mm), len(mm), d(lam), d(co), d(ba), C.c_double(eps2), C.c_double(coef), C.byref(E))
        return E.value

    def friction_gradient(self, Vt, mm, lam, co, ba, eps2, coef, g=None):
        if g is None:
            g = np.zeros(3 * self.mesh.nV)
        mm = np.ascontiguousarray(mm, dtype=np.int32); vt = self._soa(Vt)
        lam, co, ba = (np.ascontiguousarray(x, dtype=np.float64) for x in (lam, co, ba))
        lib().orc_friction_gradient(C.byref(self.s), d(vt), i(mm), len(mm), d(lam), d(co), d(ba), C.c_double(eps2), C.c_double(coef), d(g))
        return g

    def friction_pair_hessian(self, Vt, mm4, lam, co, ba, eps2, coef, project=1):
        H = np.empty(144); nv = C.c_int()
        mm4 = np.ascontiguousarray(mm4, dtype=np.int32); vt = self._soa(Vt)
        co, ba = np.ascontiguousarray(co, dtype=np.float64), np.ascontiguousarray(ba, dtype=np.float64)
        lib().orc_friction_pair_hessian(C.byref(self.s), d(vt), i(mm4), C.c_double(lam), d(co), d(ba), C.c_double(eps2), C.c_double(coef), project, d(H), C.byref(nv))
        return H.reshape(12, 12), nv.value

    def friction_hessian_csr(self, Vt, mm, lam, co, ba, eps2, coef, ia, ja, base, projectDBC=1, a=None, nthreads=1):
        ia = np.ascontiguousarray(ia, dtype=np.int32); ja = np.ascontiguousarray(ja, dtype=np.int32)
        if a is None:
            a = np.zeros(ja.size)
        mm = np.ascontiguousarray(mm, dtype=np.int32); vt = self._soa(Vt)
        lam, co, ba = (np.ascontiguousarray(x, dtype=np.float64) for x in (lam, co, ba))
        lib().orc_friction_hessian_csr(C.byref(self.s), d(vt), i(mm), len(mm), d(lam), d(co), d(ba), C.c_double(eps2), C.c_double(coef), projectDBC,
                                       i(ia), i(ja), base, d(a), nthreads)
        return a

    def pair_hessian(self, mm4, dHat, kappa):
        H = np.empty(144); nv = C.c_int()
        mm4 = np.ascontiguousarray(mm4, dtype=np.int32)
        lib().orc_barrier_pair_hessian(C.byref(self.s), i(mm4), C.c_double(dHat), C.c_double(kappa), d(H), C.byref(nv))
        return H.reshape(12, 12), nv.value


# ---- CCD (Tight-Inclusion restatement) -----------------------------------------------------------------------------
class OrcGrid(C.Structure):
    _fields_ = [("lo", C.c_double * 3), ("inv_h", C.c_double), ("count", C.c_int * 3)]


def ti(kind, x0, x1, err, ms, tol=1e-6, max_t=1.0, max_itr=1000000, no_zero_toi=1):
    x0 = np.ascontiguousarray(x0, dtype=np.float64).ravel(); x1 = np.ascontiguousarray(x1, dtype=np.float64).ravel()
    err = np.ascontiguousarray(err, dtype=np.float64)
    toi, ot = C.c_double(), C.c_double()
    fn = lib().orc_ti_vf if kind == "vf" else lib().orc_ti_ee
    hit = fn(d(x0), d(x1), d(err), C.c_double(ms), C.c_double(tol), C.c_double(max_t), int(max_itr), int(no_zero_toi), C.byref(toi), C.byref(ot))
    return bool(hit), toi.value, ot.value


TI_EXITS = ("exhausted", "k1", "k2", "skip", "max_itr", "depth60", "level_cap", "unfinished")


def ti_trace(kind, x0, x1, err, tol=1e-6, max_t=1.0, trip_cap=1000, box_cap=1 << 24, level_cap=0):
    """One pair as the narrow phase runs it (ms from the initial distance, max_itr 1e6, no_zero_toi, the ms = 0 retry), traced.
    level_cap > 0 emulates level buffers that return the per-level estimate when a level outgrows them.
    Returns (r, toi, trace): r = -1 zero distance / 0 no impact / 1 impact."""
    x0 = np.ascontiguousarray(x0, dtype=np.float64).ravel(); x1 = np.ascontiguousarray(x1, dtype=np.float64).ravel()
    err = np.ascontiguousarray(err, dtype=np.float64)
    toi = C.c_double()
    oi = np.zeros(17, dtype=np.int64); od = np.zeros(3)
    lib().orc_ti_debug_level_cap(C.c_longlong(int(level_cap)))
    try:
        r = lib().orc_ti_trace(int(kind == "vf"), d(x0), d(x1), d(err), C.c_double(tol), C.c_double(max_t), C.c_longlong(int(trip_cap)),
                               C.c_longlong(int(box_cap)), C.byref(toi), oi.ctypes.data_as(C.POINTER(C.c_longlong)), d(od))
    finally:
        lib().orc_ti_debug_level_cap(C.c_longlong(0))
    tr = dict(exits={TI_EXITS[e]: int(oi[e]) for e in range(8)}, last_exit=TI_EXITS[oi[8]] if oi[8] >= 0 else None, unfinished=bool(oi[9]),
              retry=bool(oi[10]), levels=int(oi[11]), width=int(oi[12]), boxes=int(oi[13]), trips=[int(x) for x in oi[14:17]],
              ms=float(od[0]), tolerance=float(od[1]), t_max=float(od[2]))
    tr["early_outs"] = tr["exits"]["max_itr"] + tr["exits"]["depth60"] + tr["exits"]["level_cap"]
    return int(r), toi.value, tr


def ti_error(V_soa, nV, p=None):
    V_soa = np.ascontiguousarray(V_soa, dtype=np.float64)
    evf, eee = np.empty(3), np.empty(3)
    lib().orc_ti_error(d(V_soa), nV, d(np.ascontiguousarray(p, dtype=np.float64)) if p is not None else None, d(evf), d(eee))
    return evf, eee


def grid_swept(surf, p, alpha, h):
    g = OrcGrid()
    a = C.c_double(alpha)
    p = np.ascontiguousarray(p, dtype=np.float64)
    lib().orc_grid_swept(C.byref(surf.s), d(p), C.byref(a), C.c_double(h), C.byref(g))
    return g, a.value


def ccd_partial(surf, p, cand, tol, evf, eee, alpha, nthreads=1):
    p = np.ascontiguousarray(p, dtype=np.float64); cand = np.ascontiguousarray(cand, dtype=np.int32)
    a = C.c_double(alpha)
    z = lib().orc_ccd_partial(C.byref(surf.s), d(p), i(cand), len(cand), C.c_double(tol), d(np.ascontiguousarray(evf)), d(np.ascontiguousarray(eee)), C.byref(a), nthreads)
    return a.value, z


def ccd_full(surf, p, grid, alpha_grid, tol, evf, eee, alpha, nthreads=1):
    p = np.ascontiguousarray(p, dtype=np.float64)
    a = C.c_double(alpha)
    n = C.c_longlong()
    z = lib().orc_ccd_full(C.byref(surf.s), d(p), C.byref(grid), C.c_double(alpha_grid), C.c_double(tol), d(np.ascontiguousarray(evf)), d(np.ascontiguousarray(eee)),
                           C.byref(a), C.byref(n), nthreads)
    return a.value, z, n.value


def ccd_full_hashed(surf, p, alpha, voxel_size, tol, evf, eee, nthreads=1):
    p = np.ascontiguousarray(p, dtype=np.float64)
    a = C.c_double(alpha)
    n = C.c_longlong()
    z = lib().orc_ccd_full_hashed(C.byref(surf.s), d(p), C.byref(a), C.c_double(voxel_size), C.c_double(tol), d(np.ascontiguousarray(evf)), d(np.ascontiguousarray(eee)),
                                  C.byref(n), nthreads)
    return a.value, z, n.value


def orient3d(a, b, c, d_, exact=False):
    a, b, c, d_ = (np.ascontiguousarray(x, dtype=np.float64) for x in (a, b, c, d_))
    f = lib().orc_orient3d_exact if exact else lib().orc_orient3d
    return int(f(d(a), d(b), d(c), d(d_)))


ORIENT3D_TRACE_FIELDS = ("cda", "dab", "abc", "bcd", "pair_sum", "adet", "bdet", "cdet", "ddet", "running_sum", "det")


def orient3d_trace(a, b, c, d_):
    """(sign, filter decided, {component counts of the exact stage}; empty when the filter decided)"""
    a, b, c, d_ = (np.ascontiguousarray(x, dtype=np.float64) for x in (a, b, c, d_))
    info = np.zeros(12, np.int32)
    s = int(lib().orc_orient3d_trace(d(a), d(b), d(c), d(d_), i(info)))
    return s, bool(info[0]), ({} if info[0] else dict(zip(ORIENT3D_TRACE_FIELDS, info[1:].tolist())))


def seg_tri_intersect(e0, e1, t0, t1, t2):
    v = [np.ascontiguousarray(x, dtype=np.float64) for x in (e0, e1, t0, t1, t2)]
    return int(lib().orc_seg_tri_intersect(*[d(x) for x in v]))


def seg_tri_trace(e0, e1, t0, t1, t2):
    """(decision, exit: 0 coplanar endpoint / 1 one side / 2 solved, rank, uvt) -- rank and uvt only for exit 2"""
    v = [np.ascontiguousarray(x, dtype=np.float64) for x in (e0, e1, t0, t1, t2)]
    ex, rk, uvt = C.c_int(), C.c_int(-1), np.full(3, np.nan)
    r = int(lib().orc_seg_tri_trace(*[d(x) for x in v], C.byref(ex), C.byref(rk), d(uvt)))
    return r, ex.value, (rk.value if ex.value == 2 else None), (uvt if ex.value == 2 else None)


# ---- kinematic mesh obstacles: MeshCO<3> (oracle/meshco.cpp) ----------------------------------------------------------------------
class OrcObstacle(C.Structure):
    _fields_ = [("nV", C.c_int), ("V", _dp), ("nE", C.c_int), ("E", _ip), ("nF", C.c_int), ("F", _ip)]


class Obstacle:
    """A triangle mesh without degrees of freedom next to a Surf: V (nVo x 3), E (nEo x 2), F (nFo x 3), the obstacle's own indices."""

    def __init__(self, surf, V, E, F):
        self.surf = surf
        self.Vo = np.ascontiguousarray(np.asarray(V, dtype=np.float64).T).ravel()
        self.E = np.ascontiguousarray(E, dtype=np.int32).ravel()
        self.F = np.ascontiguousarray(np.asarray(F, dtype=np.int32).T).ravel()
        self.nV, self.nE, self.nF = len(V), len(E), len(F)
        self.o = OrcObstacle(self.nV, d(self.Vo), self.nE, i(self.E), self.nF, i(self.F))

    def constraint_set(self, dHat, nthreads=1, cap=1 << 18):
        mm = np.empty((cap, 4), dtype=np.int32); pa = np.empty((cap, 4), dtype=np.int32); pe = np.empty((cap, 2), dtype=np.int32)
        cand = np.empty((4 * cap, 2), dtype=np.int32)
        nC, nP, nK = C.c_int(), C.c_int(), C.c_int()
        rc = lib().orc_meshco_constraint_set(C.byref(self.surf.s), C.byref(self.o), C.c_double(dHat), cap, i(mm), C.byref(nC), cap, i(pa), i(pe), C.byref(nP),
                                             4 * cap, i(cand), C.byref(nK), nthreads)
        assert rc == 0, "oracle constraint-set capacity exceeded"
        return mm[:nC.value].copy(), pa[:nP.value].copy(), pe[:nP.value].copy(), cand[:nK.value].copy()

    def to_merged(self, mm, pe):
        """MeshCO entries -> self-contact entries over the merged numbering (what the GPU library reports)"""
        mm = np.ascontiguousarray(mm, dtype=np.int32); pe = np.ascontiguousarray(pe, dtype=np.int32)
        out = np.empty_like(mm); pe_out = np.empty_like(pe)
        lib().orc_meshco_to_merged(self.surf.mesh.nV, self.surf.SE.size // 2, i(mm), len(mm), i(out), i(pe), len(pe), i(pe_out))
        return out, pe_out

    def _sets(self, mm, pa, pe):
        return tuple(np.ascontiguousarray(x, dtype=np.int32) for x in (mm, pa, pe))

    def energy(self, mm, pa, pe, dHat, kappa):
        mm, pa, pe = self._sets(mm, pa, pe)
        E = C.c_double()
        bad = lib().orc_meshco_energy(C.byref(self.surf.s), C.byref(self.o), i(mm), len(mm), i(pa), i(pe), len(pa), C.c_double(dHat), C.c_double(kappa), C.byref(E))
        return E.value, bad

    def gradient(self, mm, pa, pe, dHat, kappa, g=None):
        mm, pa, pe = self._sets(mm, pa, pe)
        if g is None:
            g = np.zeros(3 * self.surf.mesh.nV)
        lib().orc_meshco_gradient(C.byref(self.surf.s), C.byref(self.o), i(mm), len(mm), i(pa), i(pe), len(pa), C.c_double(dHat), C.c_double(kappa), d(g))
        return g

    def hessian_csr(self, mm, pa, pe, dHat, kappa, ia, ja, base, projectDBC=1, a=None, nthreads=1):
        mm, pa, pe = self._sets(mm, pa, pe)
        ia = np.ascontiguousarray(ia, dtype=np.int32); ja = np.ascontiguousarray(ja, dtype=np.int32)
        if a is None:
            a = np.zeros(ja.size)
        lib().orc_meshco_hessian_csr(C.byref(self.surf.s), C.byref(self.o), i(mm), len(mm), i(pa), i(pe), len(pa), C.c_double(dHat), C.c_double(kappa), projectDBC,
                                     i(ia), i(ja), base, d(a), nthreads)
        return a

    def ccd_partial(self, p, cand, tol, evf, eee, alpha, ee_as_vf=1, nthreads=1):
        p = np.ascontiguousarray(p, dtype=np.float64); cand = np.ascontiguousarray(cand, dtype=np.int32)
        a = C.c_double(alpha)
        z = lib().orc_meshco_ccd_partial(C.byref(self.surf.s), C.byref(self.o), d(p), i(cand), len(cand), C.c_double(tol), d(np.ascontiguousarray(evf)),
                                         d(np.ascontiguousarray(eee)), ee_as_vf, C.byref(a), nthreads)
        return a.value, z

    def ccd_full(self, p, tol, evf, eee, alpha, ee_as_vf=1, nthreads=1):
        p = np.ascontiguousarray(p, dtype=np.float64)
        a = C.c_double(alpha); n = C.c_longlong()
        z = lib().orc_meshco_ccd_full(C.byref(self.surf.s), C.byref(self.o), d(p), C.c_double(tol), d(np.ascontiguousarray(evf)), d(np.ascontiguousarray(eee)), ee_as_vf,
                                      C.byref(a), C.byref(n), nthreads)
        return a.value, z, n.value
